// abrb_host.hpp — host-side preparation of the kernel constants from the C-ABI structs.
// Pure C++ (no CUDA): shared by the library (api.cu) and by the CPU-side unit-test shim (tests/hostsim).
#pragma once
#include <cmath>
#include <cstring>
#include <string>

#include "../../include/abrb.h"
#include "abrb_osc.cuh"

namespace abrb {

struct ChainHost {
  int n = 0;
  bool ortho = true;
  double G0[12], L0[12], Bf[kMaxJoints][12], BA[kMaxJoints][12];
  double Wp[kMaxJoints + 1][3], Wos[kMaxJoints][3], gp[kMaxJoints + 1][3], gos[kMaxJoints][3];
};

inline void aff_mul_h(const double *X, const double *C, double *o) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) o[r * 4 + c] = X[r * 4] * C[c] + X[r * 4 + 1] * C[4 + c] + X[r * 4 + 2] * C[8 + c];
    o[r * 4 + 3] = X[r * 4] * C[3] + X[r * 4 + 1] * C[7] + X[r * 4 + 2] * C[11] + X[r * 4 + 3];
  }
}

inline bool block_orthonormal(const double *X) {
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double s = 0;
      for (int r = 0; r < 3; ++r) s += X[r * 4 + a] * X[r * 4 + b];
      if (std::fabs(s - (a == b ? 1.0 : 0.0)) > 1e-12) return false;
    }
  return true;
}

// returns an error message or empty string
inline std::string chain_from_desc(const abrb_chain_desc &d, ChainHost &h) {
  if (d.n_joints < 1 || d.n_joints > kMaxJoints) return "n_joints out of range [1, ABRB_MAX_JOINTS]";
  if (d.n_links != d.n_joints + 1) return "n_links must equal n_joints + 1";
  const int n = h.n = d.n_joints;
  std::memcpy(h.L0, d.L0, sizeof h.L0);
  aff_mul_h(d.L0, d.A[0], h.G0);
  h.ortho = block_orthonormal(d.L0) && block_orthonormal(d.E);
  for (int i = 0; i < n; ++i) {
    h.ortho = h.ortho && block_orthonormal(d.A[i]) && block_orthonormal(d.B[i]);
    std::memcpy(h.Bf[i], d.B[i], sizeof h.Bf[i]);
    aff_mul_h(d.B[i], i < n - 1 ? d.A[i + 1] : d.E, h.BA[i]);
  }
  for (int l = 0; l <= n; ++l)
    for (int c = 0; c < 3; ++c) {
      h.Wp[l][c] = d.link_inertia[l][c];
      h.gp[l][c] = d.link_inertia[l][c] * d.gravity[c];
    }
  for (int k = 0; k < n; ++k)
    for (int c = 0; c < 3; ++c) {
      double s = 0, sg = 0;
      for (int l = k + 1; l <= n; ++l) {
        s += d.link_inertia[l][3 + c];
        sg += d.link_inertia[l][3 + c] * d.gravity[3 + c];
      }
      h.Wos[k][c] = s;
      h.gos[k][c] = sg;
    }
  for (int i = 0; i < 12; ++i)
    if (!std::isfinite(h.G0[i])) return "non-finite chain constant";
  return "";
}

template <typename T, int N>
inline void fill_chain(const ChainHost &h, ChainK<T, N> &P) {
  for (int i = 0; i < 12; ++i) {
    P.G0[i] = T(h.G0[i]);
    P.L0[i] = T(h.L0[i]);
  }
  for (int k = 0; k < N; ++k) {
    for (int i = 0; i < 12; ++i) {
      P.Bf[k][i] = T(h.Bf[k][i]);
      P.BA[k][i] = T(h.BA[k][i]);
    }
    for (int c = 0; c < 3; ++c) {
      P.Wos[k][c] = T(h.Wos[k][c]);
      P.gos[k][c] = T(h.gos[k][c]);
    }
  }
  for (int l = 0; l <= N; ++l)
    for (int c = 0; c < 3; ++c) {
      P.Wp[l][c] = T(h.Wp[l][c]);
      P.gp[l][c] = T(h.gp[l][c]);
    }
}

inline int parse_frame(int n, const char *name) {
  // reference: "link#", "joint#", "EE" (arms/ur5/config.py:301-337); anything else is invalid
  if (name == nullptr) return ABRB_EFRAME;
  if (std::strcmp(name, "EE") == 0) return 2 * n + 1;
  auto num = [](const char *s, int &v) {
    if (*s == 0) return false;
    v = 0;
    for (; *s; ++s) {
      if (*s < '0' || *s > '9') return false;
      v = v * 10 + (*s - '0');
      if (v > 1000) return false;
    }
    return true;
  };
  int v;
  if (std::strncmp(name, "link", 4) == 0 && num(name + 4, v) && v <= n) return v;
  if (std::strncmp(name, "joint", 5) == 0 && num(name + 5, v) && v < n) return n + 1 + v;
  return ABRB_EFRAME;
}

inline std::string check_null(int n, const abrb_null_params &z) {
  if (z.kind != ABRB_NULL_DAMPING && z.kind != ABRB_NULL_RESTING && z.kind != ABRB_NULL_AVOID &&
      z.kind != ABRB_NULL_JOINT_LIMITS)
    return "unknown secondary controller kind";
  if (z.kind == ABRB_NULL_AVOID && (z.n_obstacles < 0 || z.n_obstacles > ABRB_MAX_OBSTACLES))
    return "n_obstacles out of range";
  (void)n;
  return "";
}

template <typename T, int N>
inline void fill_null(const abrb_null_params &z, NullK<T, N> &Z) {
  Z.kind = z.kind;
  Z.n_obs = z.kind == ABRB_NULL_AVOID ? z.n_obstacles : 0;
  Z.rest_mask = 0;
  Z.pad_ = 0;
  Z.kp = T(z.kp);
  Z.kv = T(z.kv);
  for (int k = 0; k < N; ++k) {
    Z.rest[k] = T(z.rest_angles[k]);
    if (z.rest_mask[k]) Z.rest_mask |= 1u << k;
  }
  Z.threshold = T(z.threshold);
  Z.gain = T(z.gain);
  Z.maximum = T(z.maximum);
  for (int o = 0; o < kMaxObstacles; ++o)
    for (int c = 0; c < 4; ++c) Z.obs[o][c] = o < Z.n_obs ? T(z.obstacles[o][c]) : T(0);
  if (z.kind == ABRB_NULL_JOINT_LIMITS) {  // shares rest[] / obs[] / rest_mask (NullK, abrb_osc.cuh)
    Z.rest_mask = 0;
    for (int k = 0; k < N; ++k) {
      const bool no_lo = z.limit_min[k] != z.limit_min[k], no_hi = z.limit_max[k] != z.limit_max[k];  // NaN
      Z.rest[k] = T(z.limit_min[k]);
      Z.obs[k >> 2][k & 3] = T(z.limit_max[k]);
      Z.obs[2 + (k >> 2)][k & 3] = T(z.limit_torque[k]);
      if (z.limit_cross_zero[k]) Z.rest_mask |= 1u << k;
      if (z.limit_gradient[k]) Z.rest_mask |= 1u << (8 + k);
      if (no_lo) Z.rest_mask |= 1u << (16 + k);
      if (no_hi) Z.rest_mask |= 1u << (24 + k);
    }
  }
}

inline std::string check_osc(int n, const abrb_osc_params &p) {
  if (p.orientation_algorithm != 0 && p.orientation_algorithm != 1)
    return "Invalid algorithm number for calculating orientation error";
  if (p.n_null < 0 || p.n_null > ABRB_MAX_NULL) return "n_null out of range";
  if (!(p.kv != 0.0)) return "kv must be non-zero";
  for (int i = 0; i < p.n_null; ++i) {
    std::string e = check_null(n, p.null[i]);
    if (!e.empty()) return e;
  }
  return "";
}

// Whether an OSC call on an n-joint chain may run the plain instantiation of osc_eval (PLAIN = true, abrb_osc.cuh):
// plain task-space control of the end effector with gravity and Coriolis compensation.  That is no secondary
// controller, no target velocity, no integrator (ki == 0, so no integrated-error array), the EE frame, use_g and use_C,
// and every one of the `kd` task rows the kernel is built for controlled (x, y, z for kd = 3; all six for kd = 6).
// Everything else runs the general instantiation.
inline bool osc_plain(const abrb_osc_params &p, int n, int frame, int kd, bool has_tv, bool has_ierr) {
  if (p.n_null != 0 || has_tv || has_ierr || frame != 2 * n + 1 || !p.use_g || !p.use_C) return false;
  for (int r = 0; r < 6; ++r)
    if ((p.ctrlr_dof[r] != 0) != (r < kd)) return false;
  return true;
}

template <typename T, int N>
inline void fill_osc(const abrb_osc_params &p, int frame, const double *x_off, OscK<T, N> &O) {
  O.kp = T(p.kp);
  O.ko = T(p.ko);
  O.kv = T(p.kv);
  O.ki = T(p.ki);
  // sat_gain / scale (identical expressions in the reference, osc.py:112-115), evaluated in double
  O.lim_xyz = p.use_vmax ? T(p.vmax[0] / p.kp * p.kv) : T(0);
  O.lim_abg = p.use_vmax ? T(p.vmax[1] / p.ko * p.kv) : T(0);
  O.thr = T(p.mx_threshold);
  for (int c = 0; c < 3; ++c) O.xoff[c] = x_off ? T(x_off[c]) : T(0);
  O.dof_mask = 0;
  for (int r = 0; r < 6; ++r)
    if (p.ctrlr_dof[r]) O.dof_mask |= 1u << r;
  O.use_vmax = p.use_vmax;
  O.use_g = p.use_g;
  O.use_C = p.use_C;
  O.alg = p.orientation_algorithm;
  O.n_null = p.n_null;
  O.frame = frame;
  for (int i = 0; i < kMaxNull; ++i) {
    if (i < p.n_null) {
      fill_null<T, N>(p.null[i], O.nul[i]);
    } else {
      std::memset(&O.nul[i], 0, sizeof O.nul[i]);
    }
  }
}

}  // namespace abrb
