// abrb_dual.cuh — forward-mode dual numbers for the per-state templates (value plus one tangent).
//
// Instantiating walk / dynamics_Mg / chol / the solves / forward_dynamics_state / plant_step on Dual<T> gives the exact
// directional derivative of every output along the tangent the inputs were seeded with (DESIGN.md S3.6).  Comparisons
// look at the value only, so every branch of the real code (chol's pivot test, walk's frame tests) is taken exactly as
// in the real evaluation.  The elementary functions compute the value with the real routine of abrb_math.cuh and the
// tangent from its exact derivative.
#pragma once
#include <type_traits>

#include "abrb_math.cuh"

namespace abrb {

template <typename T>
struct Dual {
  T v, d;
  Dual() = default;
  ABRB_HD Dual(T v_, T d_) : v(v_), d(d_) {}
  template <typename U, typename = typename std::enable_if<std::is_arithmetic<U>::value>::type>
  ABRB_HD Dual(U x) : v(T(x)), d(T(0)) {}  // a constant: zero tangent

  // hidden friends: a real operand converts to a constant
  friend ABRB_HD Dual operator+(Dual a, Dual b) { return Dual(a.v + b.v, a.d + b.d); }
  friend ABRB_HD Dual operator-(Dual a, Dual b) { return Dual(a.v - b.v, a.d - b.d); }
  friend ABRB_HD Dual operator-(Dual a) { return Dual(-a.v, -a.d); }
  friend ABRB_HD Dual operator*(Dual a, Dual b) { return Dual(a.v * b.v, a.v * b.d + a.d * b.v); }
  friend ABRB_HD Dual operator/(Dual a, Dual b) {
    const T r = a.v / b.v;
    return Dual(r, (a.d - r * b.d) / b.v);
  }
  friend ABRB_HD Dual &operator+=(Dual &a, Dual b) { return a = a + b; }
  friend ABRB_HD Dual &operator-=(Dual &a, Dual b) { return a = a - b; }
  friend ABRB_HD Dual &operator*=(Dual &a, Dual b) { return a = a * b; }
  friend ABRB_HD bool operator<(Dual a, Dual b) { return a.v < b.v; }
  friend ABRB_HD bool operator>(Dual a, Dual b) { return a.v > b.v; }
  friend ABRB_HD bool operator<=(Dual a, Dual b) { return a.v <= b.v; }
  friend ABRB_HD bool operator>=(Dual a, Dual b) { return a.v >= b.v; }
  friend ABRB_HD bool operator==(Dual a, Dual b) { return a.v == b.v; }
  friend ABRB_HD bool operator!=(Dual a, Dual b) { return a.v != b.v; }
};

template <typename T>
ABRB_HD void sincos_t(Dual<T> x, Dual<T> *s, Dual<T> *c) {
  T sv, cv;
  sincos_t(x.v, &sv, &cv);
  *s = Dual<T>(sv, cv * x.d);
  *c = Dual<T>(cv, -sv * x.d);
}
template <typename T>
ABRB_HD Dual<T> inv_sqrt_t(Dual<T> x) {  // d(x^-1/2) = -1/2 x^-3/2 dx
  const T y = inv_sqrt_t(x.v);
  return Dual<T>(y, T(-0.5) * y * y * y * x.d);
}
template <typename T>
ABRB_HD Dual<T> sqrt_t(Dual<T> x) {
  const T y = sqrt_t(x.v);
  return Dual<T>(y, T(0.5) * x.d / y);
}
template <typename T>
ABRB_HD Dual<T> abs_t(Dual<T> x) {
  return x.v < T(0) ? -x : x;
}
// fmod by a constant divisor (wrap_pm_pi): the value is the real routine's, and away from the jumps (a set of measure
// zero) d fmod(x, y) = dx, so the tangent passes through unchanged
template <typename T>
ABRB_HD Dual<T> fmod_t(Dual<T> x, Dual<T> y) {
  return Dual<T>(fmod_t(x.v, y.v), x.d);
}

}  // namespace abrb
