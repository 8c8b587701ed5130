// abrb_path.cuh — per-row and per-step arithmetic of the batched path planner (include/abrb.h, abrb_path_*).
//
// Everything is fp64 and __host__ __device__, so tests/hostsim/plannersim.cpp runs the same code on the CPU.
// Reference: controllers/path_planners/path_planner.py:75-397 (warp, velocity search, interpolation, gradients),
// orientation.py:157-198 (the SLERP fraction) and utils/transformations.py (quaternion_from_euler, quaternion_slerp,
// quaternion_matrix, euler_from_matrix).  Each function states the NumPy expression it evaluates, in the same order.
#pragma once
#include "../../include/abrb.h"
#include "abrb_math.cuh"

namespace abrb {
namespace path {

constexpr double kEps = 4.0 * 2.220446049250313e-16;  // transformations._EPS
constexpr double kMaxCount = 268435456.0;             // 2^28: bound on every int() count (ABRB_PATH_TOO_LONG)
constexpr double kPi = 3.141592653589793;

// The warped curve: R (align_vectors((1,1,1)/sqrt3, target - start)), the distance and the start.
struct Frame {
  double R[3][3];
  double dist;
  double start[3];
};

// path_planner.py:184-192 and align_vectors (:75-97).  Returns 0 or a negative ABRB_PATH_* reason.
ABRB_HD int frame_of(const double *start, const double *target, Frame &F) {
  double d[3];
  for (int c = 0; c < 3; ++c) {
    F.start[c] = start[c];
    d[c] = target[c] - start[c];
  }
  F.dist = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (!(F.dist > 0.0) || !(F.dist < INFINITY)) return ABRB_PATH_ZERO_DISTANCE;
  const double a0 = 1.0 / sqrt(3.0);
  const double na = sqrt(a0 * a0 + a0 * a0 + a0 * a0);
  double a[3], b[3];
  for (int c = 0; c < 3; ++c) b[c] = d[c] / F.dist;
  const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  for (int c = 0; c < 3; ++c) {
    b[c] = b[c] / nb;
    a[c] = a0 / na;
  }
  const double v[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
  const double cth = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
  if (!(1.0 + cth > 0.0)) return ABRB_PATH_OPPOSITE;
  const double h = 1.0 / (1.0 + cth);
  const double V[3][3] = {{0.0, -v[2], v[1]}, {v[2], 0.0, -v[0]}, {-v[1], v[0], 0.0}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double vv = V[i][0] * V[0][j] + V[i][1] * V[1][j] + V[i][2] * V[2][j];
      F.R[i][j] = ((i == j ? 1.0 : 0.0) + V[i][j]) + vv * h;
    }
  return 0;
}

// warped_xyz[i] = R . ((1/sqrt3) step(t_i) dist) + start   (path_planner.py:202-205)
ABRB_HD void warp_point(const Frame &F, const double *table, int i, double *w) {
  const double s3 = 1.0 / sqrt(3.0);
  double p[3];
  for (int c = 0; c < 3; ++c) p[c] = s3 * table[3 * i + c] * F.dist;
  for (int r = 0; r < 3; ++r) w[r] = (F.R[r][0] * p[0] + F.R[r][1] * p[1] + F.R[r][2] * p[2]) + F.start[r];
}

// curve_dist_steps[i] = |warped_xyz[i] - warped_xyz[i-1]|, i >= 1
ABRB_HD double seg_len(const Frame &F, const double *table, int i) {
  double a[3], b[3];
  warp_point(F, table, i - 1, a);
  warp_point(F, table, i, b);
  const double d0 = b[0] - a[0], d1 = b[1] - a[1], d2 = b[2] - a[2];
  return sqrt(d0 * d0 + d1 * d1 + d2 * d2);
}

// np.linspace(a, b, n)[k]
ABRB_HD double linspace_at(double a, double b, int n, int k) {
  if (n > 1 && k == n - 1) return b;
  const int div = n - 1;
  const double delta = b - a;
  if (div > 0) {
    const double step = delta / div;
    if (step == 0.0) return (double(k) / div) * delta + a;
    return double(k) * step + a;
  }
  return double(k) * delta + a;
}

// One velocity ramp vel_profile.generate(va, vb): n samples (velocity_profiles.py:47-125).
struct Ramp {
  int kind, n;
  double va, vb;
  double s, u, g0, scale;  // Gaussian: sigma, mean, the unshifted first sample and the rescaling factor
};

// the argument of int() that sizes a ramp: ((vb - va) / acceleration) / dt for both kinds
ABRB_HD double ramp_count(const abrb_path_params &p, double va, double vb) {
  return ((vb - va) / p.acceleration) / p.dt;
}

ABRB_HD double gauss(const Ramp &r, double x) {
  const double z = (x - r.u) / r.s;
  return 1.0 * (1.0 / (r.s * sqrt(2.0 * kPi)) * exp(-0.5 * (z * z)));
}

ABRB_HD Ramp ramp_make(const abrb_path_params &p, double va, double vb, int n) {
  Ramp r{p.vel_kind, n, va, vb, 0.0, 0.0, 0.0, 0.0};
  if (p.vel_kind == ABRB_VEL_GAUSSIAN) {
    r.s = 1.0 / ((vb - va) * sqrt(kPi * 2.0));
    r.u = p.n_sigma * r.s;
    r.g0 = gauss(r, linspace_at(0.0, r.u, n, 0));
    r.scale = (vb - va) / (gauss(r, linspace_at(0.0, r.u, n, n - 1)) - r.g0);
  }
  return r;
}

// vel_profile[k]
ABRB_HD double ramp_at(const Ramp &r, int k) {
  if (r.kind == ABRB_VEL_LINEAR) return linspace_at(r.va, r.vb, r.n, k);
  return (gauss(r, linspace_at(0.0, r.u, r.n, k)) - r.g0) * r.scale + r.va;
}

// Reduction order of the two phases' sums (curve length, ramp distances): element i goes to partial (i - lo) % 32,
// each partial sums its elements in ascending order, and the 32 partials combine in an xor butterfly (16, 8, 4, 2, 1).
// On the device the partials are the lanes of one warp (kernels.cu, WarpSum); HostSum replays the same order.
struct HostSum {
  template <class F>
  double operator()(int lo, int n, F f) const {
    double acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.0;
    for (int i = lo; i < n; ++i) acc[(i - lo) % 32] += f(i);
    for (int off = 16; off > 0; off >>= 1) {
      double nx[32];
      for (int l = 0; l < 32; ++l) nx[l] = acc[l] + acc[l ^ off];
      for (int l = 0; l < 32; ++l) acc[l] = nx[l];
    }
    return acc[0];
  }
};

// int(x) of a count, with the rejections the reference meets as an exception or a NaN row
ABRB_HD int count_of(double x, int min_count, int &out) {
  if (!(x < kMaxCount)) return ABRB_PATH_TOO_LONG;
  if (!(x >= double(min_count))) return ABRB_PATH_SHORT_RAMP;
  out = int(x);
  return 0;
}

// Phase 1 for one row (path_planner.py:144-302): the curve length and the max_v search.  Returns S (> 0) or a negative
// ABRB_PATH_* reason; fills rec.
template <class Sum>
ABRB_HD int64_t plan_row(const abrb_path_params &p, const double *table, const double *start, const double *target,
                         double vmax, double v0, double v1, abrb_path_rec &rec, const Sum &sum) {
  Frame F;
  int rc = frame_of(start, target, F);
  if (rc) return rc;
  const double curve = sum(1, p.n_points, [&](int i) { return seg_len(F, table, i); });
  const bool s_spec = v0 == vmax, e_spec = v1 == vmax;
  // starting_dist / ending_dist: "None" until first computed; a ramp is regenerated while its distance is None or
  // non-zero (path_planner.py:153-163, 247-269), so the [v dt] special case keeps its distance 0 throughout
  bool s_none = !s_spec, e_none = !e_spec;
  double sd = 0.0, ed = 0.0, max_v = vmax;
  int ns = 1, ne = 1, nc = 0;
  for (;;) {
    if (max_v <= 0.0) return ABRB_PATH_NO_VELOCITY;
    if (s_none || sd != 0.0) {
      if ((rc = count_of(ramp_count(p, v0, max_v), 2, ns))) return rc;
      const Ramp r = ramp_make(p, v0, max_v, ns);
      sd = sum(0, ns, [&](int k) { return ramp_at(r, k) * p.dt; });
      s_none = false;
    }
    if (e_none || ed != 0.0) {
      if ((rc = count_of(ramp_count(p, v1, max_v), 2, ne))) return rc;
      const Ramp r = ramp_make(p, v1, max_v, ne);
      const int n = ne;
      ed = sum(0, ne, [&](int k) { return ramp_at(r, n - 1 - k) * p.dt; });
      e_none = false;
    }
    if (curve > sd + ed) {
      const double remaining = curve - (ed + sd);
      if ((rc = count_of(remaining / max_v / p.dt, 0, nc))) return rc;
      break;
    }
    if (curve == sd + ed) {
      nc = 0;
      break;
    }
    max_v -= 0.1;
  }
  rec.max_v = max_v;
  rec.n_start = ns;
  rec.n_const = nc;
  rec.n_end = ne;
  rec.flags = (s_spec ? 1 : 0) | (e_spec ? 2 : 0);
  return int64_t(ns) + nc + ne;
}

// The two ramps of a planned row.
struct Profile {
  Ramp start, end;
  abrb_path_rec rec;
  double v0, v1, dt;
};

ABRB_HD Profile profile_of(const abrb_path_params &p, const abrb_path_rec &rec, double v0, double v1) {
  return Profile{ramp_make(p, v0, rec.max_v, rec.n_start), ramp_make(p, v1, rec.max_v, rec.n_end), rec, v0, v1, p.dt};
}

// stacked_vel_profile[j] * dt, the increment of path_steps = cumsum(stacked_vel_profile * dt)  (path_planner.py:316)
ABRB_HD double step_at(const Profile &P, int j) {
  double v;
  if (j < P.rec.n_start) {
    v = (P.rec.flags & 1) ? P.v0 * P.dt : ramp_at(P.start, j);
  } else if (j < P.rec.n_start + P.rec.n_const) {
    v = P.rec.max_v;
  } else {
    const int e = j - P.rec.n_start - P.rec.n_const;
    v = (P.rec.flags & 2) ? P.v1 * P.dt : ramp_at(P.end, P.rec.n_end - 1 - e);
  }
  return v * P.dt;
}

// scipy interp1d(arc, xyz, kind="linear", fill_value="extrapolate")(s): searchsorted(side="left") clipped to
// [1, P-1], then ((s - x_lo)/(x_hi - x_lo)) y_hi + ((x_hi - s)/(x_hi - x_lo)) y_lo
ABRB_HD void interp(const double *arc, const double *xyz, int P, double s, double *y) {
  int lo = 0, hi = P;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (arc[m] < s)
      lo = m + 1;
    else
      hi = m;
  }
  const int i = lo < 1 ? 1 : (lo > P - 1 ? P - 1 : lo);
  const double xl = arc[i - 1], xh = arc[i];
  const double a = (s - xl) / (xh - xl), b = (xh - s) / (xh - xl);
  for (int c = 0; c < 3; ++c) y[c] = a * xyz[3 * i + c] + b * xyz[3 * (i - 1) + c];
}

// np.gradient(f, dt) (edge_order=1) at step k of S, given f[k-1], f[k], f[k+1] (unused ends ignored)
ABRB_HD double gradient_at(double fm, double f0, double fp, int k, int S, double dt) {
  if (k == 0) return (fp - f0) / dt;
  if (k == S - 1) return (f0 - fm) / dt;
  return (fp - fm) / (2.0 * dt);
}

// ------------------------------------------------------------------------------------------------- orientation
// transformations._NEXT_AXIS = [1, 2, 0, 1]
ABRB_HD int next_axis(int i) { return (i + 1) % 3; }

// transformations.quaternion_from_euler(ai, aj, ak, axes), axes = (firstaxis, parity, repetition, frame); q = (w,x,y,z)
ABRB_HD void quat_from_euler(double ai, double aj, double ak, const int32_t *axes, double *q) {
  const int fa = axes[0], par = axes[1], rep = axes[2], frm = axes[3];
  const int i = fa + 1;
  const int j = next_axis(i + par - 1) + 1;
  const int k = next_axis(i - par) + 1;
  if (frm) {
    const double t = ai;
    ai = ak;
    ak = t;
  }
  if (par) aj = -aj;
  ai /= 2.0;
  aj /= 2.0;
  ak /= 2.0;
  const double ci = cos(ai), si = sin(ai), cj = cos(aj), sj = sin(aj), ck = cos(ak), sk = sin(ak);
  const double cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  if (rep) {
    q[0] = cj * (cc - ss);
    q[i] = cj * (cs + sc);
    q[j] = sj * (cc + ss);
    q[k] = sj * (cs - sc);
  } else {
    q[0] = cj * cc + sj * ss;
    q[i] = cj * sc - sj * cs;
    q[j] = cj * ss + sj * cc;
    q[k] = cj * cs - sj * sc;
  }
  if (par) q[j] *= -1.0;
}

ABRB_HD double dot4(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3]; }

// transformations.unit_vector for a 4-vector
ABRB_HD void unit4(double *q) {
  const double n = sqrt(dot4(q, q));
  for (int c = 0; c < 4; ++c) q[c] /= n;
}

// transformations.quaternion_slerp(q0, q1, fraction) with q0, q1 already unit vectors
ABRB_HD void slerp(const double *q0, const double *q1, double fraction, double *out) {
  if (fraction == 0.0 || fraction == 1.0) {
    for (int c = 0; c < 4; ++c) out[c] = fraction == 0.0 ? q0[c] : q1[c];
    return;
  }
  double d = dot4(q0, q1);
  double sgn = 1.0;
  if (fabs(fabs(d) - 1.0) < kEps) {
    for (int c = 0; c < 4; ++c) out[c] = q0[c];
    return;
  }
  if (d < 0.0) {
    d = -d;
    sgn = -1.0;
  }
  const double angle = acos(d);
  if (fabs(angle) < kEps) {
    for (int c = 0; c < 4; ++c) out[c] = q0[c];
    return;
  }
  const double isin = 1.0 / sin(angle);
  const double a = sin((1.0 - fraction) * angle) * isin, b = sin(fraction * angle) * isin;
  for (int c = 0; c < 4; ++c) out[c] = q0[c] * a + (sgn * q1[c]) * b;
}

// transformations.euler_from_quaternion(q, axes) = euler_from_matrix(quaternion_matrix(q), axes)
ABRB_HD void euler_from_quat(const double *qin, const int32_t *axes, double *e) {
  double M[3][3];
  const double n = dot4(qin, qin);
  if (n < kEps) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) M[r][c] = r == c ? 1.0 : 0.0;
  } else {
    const double s = sqrt(2.0 / n);
    double q[4];
    for (int c = 0; c < 4; ++c) q[c] = qin[c] * s;
    double o[4][4];
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) o[r][c] = q[r] * q[c];
    M[0][0] = 1.0 - o[2][2] - o[3][3];
    M[0][1] = o[1][2] - o[3][0];
    M[0][2] = o[1][3] + o[2][0];
    M[1][0] = o[1][2] + o[3][0];
    M[1][1] = 1.0 - o[1][1] - o[3][3];
    M[1][2] = o[2][3] - o[1][0];
    M[2][0] = o[1][3] - o[2][0];
    M[2][1] = o[2][3] + o[1][0];
    M[2][2] = 1.0 - o[1][1] - o[2][2];
  }
  const int fa = axes[0], par = axes[1], rep = axes[2], frm = axes[3];
  const int i = fa, j = next_axis(i + par), k = next_axis(i - par + 1);
  double ax, ay, az;
  if (rep) {
    const double sy = sqrt(M[i][j] * M[i][j] + M[i][k] * M[i][k]);
    if (sy > kEps) {
      ax = atan2(M[i][j], M[i][k]);
      ay = atan2(sy, M[i][i]);
      az = atan2(M[j][i], -M[k][i]);
    } else {
      ax = atan2(-M[j][k], M[j][j]);
      ay = atan2(sy, M[i][i]);
      az = 0.0;
    }
  } else {
    const double cy = sqrt(M[i][i] * M[i][i] + M[j][i] * M[j][i]);
    if (cy > kEps) {
      ax = atan2(M[k][j], M[k][k]);
      ay = atan2(-M[k][i], cy);
      az = atan2(M[j][i], M[i][i]);
    } else {
      ax = atan2(-M[j][k], M[j][j]);
      ay = atan2(-M[k][i], cy);
      az = 0.0;
    }
  }
  if (par) {
    ax = -ax;
    ay = -ay;
    az = -az;
  }
  if (frm) {
    const double t = ax;
    ax = az;
    az = t;
  }
  e[0] = ax;
  e[1] = ay;
  e[2] = az;
}

ABRB_HD double norm3_diff(const double *a, const double *b) {
  const double d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
  return sqrt(d0 * d0 + d1 * d1 + d2 * d2);
}

// Orientation at a position p of the path (orientation.py:181-196): fraction = 1 - |p_end - p| / |p_end - p_0|, then
// Euler angles of slerp(q0, q1, fraction).  q0, q1 are the unit start and target quaternions.
ABRB_HD void orient_at(const double *q0, const double *q1, const int32_t *axes, const double *p0, const double *pe,
                       const double *p, double *e) {
  const double f = 1.0 - norm3_diff(pe, p) / norm3_diff(pe, p0);
  double q[4];
  slerp(q0, q1, f, q);
  euler_from_quat(q, axes, e);
}

// Unit quaternion of Euler angles (the planner's quat0 / quat1 before the SLERP normalises them).
ABRB_HD void unit_quat(const double *euler, const int32_t *axes, double *q) {
  quat_from_euler(euler[0], euler[1], euler[2], axes, q);
  unit4(q);
}

}  // namespace path
}  // namespace abrb
