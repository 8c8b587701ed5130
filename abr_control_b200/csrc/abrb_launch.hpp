// abrb_launch.hpp — host-side launch interface between api.cu and the per-joint-count kernel TUs.
#pragma once
#include <cuda_runtime.h>

#include "abrb_host.hpp"

namespace abrb {

struct RbdCall {
  int frame;
  const double *xoff;  // host, 3 values or nullptr
  const void *q, *dq;  // device
  int64_t B;
  abrb_rbd_out out;    // device pointers
  bool f32;
  cudaStream_t stream;
};

// Fused all-gather of the control outputs over NVLink peer memory (BASELINE config 5): the OSC kernel's epilogue stores
// every rank's rows straight into the gathered (B_total, n) array of EVERY rank (buffers mapped with CUDA IPC), so the
// exchange overlaps the arithmetic tile by tile instead of following it as a separate collective.
struct GatherArgs {
  void *peer_u[kMaxPeers];                  // base of the gathered array on each rank (own rank included)
  unsigned long long *peer_flag[kMaxPeers]; // &flags[my_rank] on each rank: receives `epoch` when all my rows are there
  int n_peer = 0;
  int self = 0;                             // this rank's index in peer_u / peer_flag
  int64_t row0 = 0;                         // first row of this rank's block in the gathered array
  unsigned long long epoch = 0;
  unsigned *cta_counter = nullptr;          // local: CTAs of this launch that have finished
};

struct OscCall {
  int frame;
  const double *xoff;
  const void *q, *dq, *target, *tv;  // device
  int target_stride, tv_stride;
  void *u, *train;
  int64_t B;
  bool f32;
  cudaStream_t stream;
  void *ierr = nullptr;  // (B, 6) integrated task-space error, in/out (device), only with ki != 0
  const GatherArgs *gather = nullptr;
  int *sched = nullptr;  // device: {next tile, CTAs done}, zero between launches (api.cu, sched_slot), or nullptr
};

struct RolloutCall {
  int frame;
  const double *xoff;
  void *q, *dq;  // device, in/out
  const void *target;
  int target_stride;
  int steps;
  double dt;
  void *q_traj, *dq_traj, *u_traj;
  int64_t B;
  bool f32;
  cudaStream_t stream;
  void *ierr = nullptr;  // (B, 6) integrated task-space error, in/out (device), only with ki != 0
};

// abrb_osc_rollout_path_*: `target` / `target_stride` hold the path, (steps, B, 6) for stride 6, (steps, 6) for 0
struct RolloutPathCall : RolloutCall {
  const void *tv = nullptr;  // path velocity, laid out like the path per tv_stride, or nullptr
  int tv_stride = 0;
  void *x_traj = nullptr;    // (steps, B, 3) or nullptr
  void *cost = nullptr;      // (B,) or nullptr
  double effort_weight = 0;
};

struct NullCall {
  const void *q, *dq;
  void *u;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// Joint (kind 0) and Floating (kind 1) controllers
struct CtrlCall {
  int kind;
  double kp, kv;
  int flag_a, flag_b;              // Joint: account_for_gravity, -   Floating: task_space, dynamic
  const void *q, *dq, *target, *tv;
  int target_stride, tv_stride;
  void *u;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

struct SlidingCall {
  double kd, lamb;
  int cartesian, frame;
  const double *xoff;  // host, 3 values or nullptr
  const void *q, *dq, *target, *tv, *ta;
  int target_stride, tv_stride, ta_stride;
  void *u, *s;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

struct IkCall {
  double max_dx, max_dr, max_dq, dt;
  int method, steps;
  const void *position, *target;
  int target_stride;
  void *pos_path, *vel_path;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_plant_rollout_*: open-loop rollout of the plant under a given torque sequence
struct PlantCall {
  int frame;
  const double *xoff;  // host, 3 values or nullptr
  void *q, *dq;        // device, in/out
  const void *u;       // (steps, B, n) for u_stride n, (steps, n) for 0
  int u_stride;
  int compensate_gravity;
  const void *path;    // (steps, B, 6) for path_stride 6, (steps, 6) for 0, or nullptr
  int path_stride;
  int steps;
  double dt, effort_weight;
  void *q_traj, *dq_traj, *u_traj, *x_traj, *cost;  // each nullptr or device
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_joint_rollout_path_* (kind kCtrlJoint) and abrb_sliding_rollout_path_* (kCtrlSliding): closed-loop rollouts
struct CtrlRolloutCall {
  int kind;
  double kp, kv;  // Joint
  int gravity;
  double kd, lamb;  // Sliding
  int cartesian;
  int frame;
  const double *xoff;           // host, 3 values or nullptr
  void *q, *dq;                 // device, in/out
  const void *path, *pv, *pa;   // (steps, B, w) for stride w, (steps, w) for 0; pv, pa may be nullptr
  int path_stride, pv_stride, pa_stride;
  int steps;
  double dt, effort_weight;
  void *q_traj, *dq_traj, *u_traj, *x_traj, *cost;  // each nullptr or device
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_forward_dynamics_* (kind 0: in = u, out = ddq) and abrb_inverse_dynamics_* (kind 1: in = ddq, out = u)
struct DynCall {
  int kind;
  const void *q, *dq, *in;
  void *out;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_inverse_dynamics_regressor_*: Yt (B, 6n, n), the transposed regressor of every state
struct RegressorCall {
  const void *q, *dq, *ddq;
  void *Yt;
  int64_t B;
  const double *gravity;  // host, 6 values (the model's)
  bool f32;
  cudaStream_t stream;
};

// abrb_forward_dynamics_derivatives_* (kind 0: in = u) and abrb_inverse_dynamics_derivatives_* (kind 1: in = ddq):
// (B, n, n) derivatives of the output with respect to q, dq and in (d_in may be nullptr)
struct DynJacCall {
  int kind;
  const void *q, *dq, *in;
  void *d_q, *d_dq, *d_in;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_plant_rollout_vjp_*: the rollout's arguments, its recorded states and the cotangents of its outputs (each
// nullptr or device) -> the cotangents of u (per trajectory), q0 and dq0
struct PlantVjpCall {
  int frame;
  const double *xoff;  // host, 3 values or nullptr
  const void *q0, *dq0, *u;
  int u_stride;
  int compensate_gravity;
  const void *path;
  int path_stride;
  int steps;
  double dt, effort_weight;
  const void *q_traj, *dq_traj;
  const void *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  void *gu, *gq0, *gdq0;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// abrb_joint_rollout_path_vjp_*: the Joint rollout's arguments, its recorded states and the cotangents of its outputs
// (each nullptr or device) -> the cotangents of the path, the path velocity and the gains (each nullptr when not
// wanted; per trajectory), q0 and dq0
struct JointVjpCall {
  double kp, kv;
  int gravity;
  int frame;
  const double *xoff;  // host, 3 values or nullptr
  const void *q0, *dq0, *path, *pv;
  int path_stride, pv_stride;
  int steps;
  double dt, effort_weight;
  const void *q_traj, *dq_traj;
  const void *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  void *g_path, *g_pv, *g_gains, *gq0, *gdq0;
  int64_t B;
  bool f32;
  cudaStream_t stream;
};

// Each returns a cudaError_t (0 = success).  Defined once per joint count in kernels.cu (-DABRB_N=<n>).
template <int N> int launch_rbd(const ChainHost &h, const RbdCall &c);
template <int N> int launch_osc(const ChainHost &h, const abrb_osc_params &p, const OscCall &c);
template <int N> int launch_rollout(const ChainHost &h, const abrb_osc_params &p, const RolloutCall &c);
template <int N> int launch_rollout_path(const ChainHost &h, const abrb_osc_params &p, const RolloutPathCall &c);
template <int N> int launch_null(const ChainHost &h, const abrb_null_params &z, const NullCall &c);
template <int N> int launch_ctrl(const ChainHost &h, const CtrlCall &c);
template <int N> int launch_sliding(const ChainHost &h, const SlidingCall &c);
template <int N> int launch_ik(const ChainHost &h, const IkCall &c);
template <int N> int launch_plant(const ChainHost &h, const PlantCall &c);
template <int N> int launch_dyn(const ChainHost &h, const DynCall &c);
template <int N> int launch_regressor(const ChainHost &h, const RegressorCall &c);
template <int N> int launch_ctrl_rollout(const ChainHost &h, const CtrlRolloutCall &c);
template <int N> int launch_dyn_jac(const ChainHost &h, const DynJacCall &c);
template <int N> int launch_plant_vjp(const ChainHost &h, const PlantVjpCall &c);
template <int N> int launch_joint_vjp(const ChainHost &h, const JointVjpCall &c);

// Path planner (abrb_path_*): independent of the joint count, compiled in the ABRB_N == 1 unit only.  Device arrays.
struct PathCall {
  abrb_path_params p;
  const double *table, *start, *target, *max_v, *v0, *v1, *so, *to;
  int64_t *lengths;   // phase 1 out, phase 2 in
  abrb_path_rec *plan;
  int64_t s_max;
  void *path;         // phase 2 out, (s_max, B, 12 or 6)
  int64_t B;
  bool f32;
  cudaStream_t stream;
};
int launch_path_plan(const PathCall &c);
int launch_path_fill(const PathCall &c);

void count_launch();

}  // namespace abrb
