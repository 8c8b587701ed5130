/*
 * abrb.h — C ABI of libabrb.so: batched rigid-body quantities and operational-space control
 *          for serial robot arms on NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for ONE hot path of abr/abr_control (SURVEY.md S8b).  Each entry
 * point states the reference interface it replaces (paths relative to the reference checkout).
 * In the reference the inner boundary is a run-time generated Cython function
 *      def autofunc_c(double q0, ..., [double dq0, ...], [double x, double y, double z]) -> ndarray
 * wrapping  void autofunc(double q0, ..., double *out)   (emitted by
 * abr_control/arms/base_config.py:125-146, loaded at :148-201), called once per joint state.
 * Here one call evaluates a whole batch of B joint states on the GPU.
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in signatures (`stream` is a cudaStream_t passed as void*,
 *     NULL = the legacy default stream);
 *   - unless the name contains `_host`, every data pointer is a DEVICE pointer on the current CUDA device,
 *     aligned to its element type (any row of a contiguous array is a valid start), row-major, batch-major: q is (B, n_joints), J is (B, 6, n_joints), M is (B, n, n) ...
 *     exactly the per-state shapes the reference returns, stacked;
 *   - the library never allocates or frees caller buffers; device-pointer calls are asynchronous with
 *     respect to the host (enqueued on `stream`); `_host` calls copy in, run, copy out and synchronise;
 *   - every function returns 0 (ABRB_OK) or a negative ABRB_E* code; abrb_last_error() gives the
 *     message for the calling thread;
 *   - handles are immutable after creation, so concurrent calls on different streams are allowed;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with ABRB_ECUDA.
 */
#ifndef ABRB_H_
#define ABRB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ABRB_VERSION 200 /* 0.2.0: integrated_error arguments, asynchronous host slots, peer-gather epilogue */
#define ABRB_MAX_JOINTS 7
#define ABRB_MAX_NULL 4
#define ABRB_MAX_OBSTACLES 16

enum {
  ABRB_OK = 0,
  ABRB_EINVAL = -1,   /* bad argument (NULL handle, B < 0, misaligned pointer, ...) */
  ABRB_EFRAME = -2,   /* reference: Exception("Invalid transformation name: ...") (arms/ur5/config.py:336-337) */
  ABRB_ESHAPE = -3,   /* n_joints / n_links outside what the library was built for */
  ABRB_EUNSUP = -4,   /* reference: NotImplementedError / Exception("Invalid algorithm number") (controllers/osc.py:190-194) */
  ABRB_ECUDA = -5,    /* CUDA runtime error (no device, launch failure, ...) */
  ABRB_ENOMEM = -6
};

/* ---------------------------------------------------------------------------------------------------
 * Arm model.  Replaces the per-arm `Config` classes' model data (arms/ur5/config.py:52-339,
 * arms/jaco2/config.py:56-356, arms/threejoint/config.py:45-223, arms/twojoint/config.py:30-181) in the
 * flattened chain form of SURVEY.md Appendix A.1:
 *     link0 = L0,  joint_i = link_i.A[i],  link_{i+1} = joint_i.Rz(q_i).B[i],  EE = link_n.E
 * All matrices are 3x4 row-major [R|t] blocks of the 4x4 homogeneous factors.  The rotation blocks are
 * NOT required to be orthonormal (Jaco2's measured frames are not; SURVEY.md S0.4).
 * ------------------------------------------------------------------------------------------------- */
typedef struct abrb_chain_desc {
  int32_t n_joints;                              /* 1 .. ABRB_MAX_JOINTS */
  int32_t n_links;                               /* must equal n_joints + 1 (link0 .. link_n) */
  double L0[12];
  double A[ABRB_MAX_JOINTS][12];
  double B[ABRB_MAX_JOINTS][12];
  double E[12];
  double link_inertia[ABRB_MAX_JOINTS + 1][6];   /* diag(m,m,m,Ixx,Iyy,Izz) of `_M_LINKS[l]` (base_config.py:625-632) */
  double gravity[6];                             /* `self.gravity`, base_config.py:123: [0,0,-9.81,0,0,0] */
} abrb_chain_desc;

typedef struct abrb_model abrb_model;

int abrb_version(void);
const char *abrb_last_error(void);
/* number of CUDA devices visible, or ABRB_ECUDA */
int abrb_device_count(void);

int abrb_model_create(const abrb_chain_desc *desc, abrb_model **out);
int abrb_model_destroy(abrb_model *m);
int abrb_model_n_joints(const abrb_model *m);
/* 1 if every constant rotation block is orthonormal to 1e-12 (selects the cross-product kernels) */
int abrb_model_is_orthonormal(const abrb_model *m);
/* Frame name -> id.  Names as in the reference: "link0".."link<n>", "joint0".."joint<n-1>", "EE".
 * Unknown names return ABRB_EFRAME (reference raises Exception, arms/ur5/config.py:336-337). */
int abrb_frame_id(const abrb_model *m, const char *name);

/* ---------------------------------------------------------------------------------------------------
 * Batched rigid-body quantities.  One call replaces, for B states at once, the reference methods
 *   Tx (base_config.py:371-392 / :739-789)     T (:338-369)          R (:287-301 / :647-676)
 *   T_inv (:394-415 / :791-837)                quaternion (:304-318) J (:249-270 / :522-592)
 *   dJ (:225-247 / :470-520)                   M (:272-285 / :594-645)
 *   g (:210-223 / :417-468)                    C (:320-336 / :678-727)
 * A NULL output pointer means "not wanted".  Frame-dependent outputs (Tx, T, R, T_inv, quat, J, dJ) are
 * for frame `frame_id` and the point `x_off` (3 host doubles, NULL = origin) inside that frame; M, g, C
 * do not depend on them.  `dq` may be NULL unless dJ or C is requested.
 * Shapes per state: Tx[3]  T[4][4]  R[3][3]  T_inv[4][4]  quat[4] (w,x,y,z)  J[6][n]  dJ[6][n]  M[n][n]
 * g[n]  C[n][n].   Unlike the reference's public wrappers nothing is rounded to float32 in the f64 variant.
 * ------------------------------------------------------------------------------------------------- */
typedef struct abrb_rbd_out {
  void *Tx, *T, *R, *T_inv, *quat, *J, *dJ, *M, *g, *C;
} abrb_rbd_out;

int abrb_rbd_eval_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q,
                      const double *dq, int64_t B, const abrb_rbd_out *out, void *stream);
int abrb_rbd_eval_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q,
                      const float *dq, int64_t B, const abrb_rbd_out *out, void *stream);
/* same, q/dq/outputs are HOST pointers; H2D + kernel + D2H + sync inside the call */
int abrb_rbd_eval_host_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q,
                           const double *dq, int64_t B, const abrb_rbd_out *out);
int abrb_rbd_eval_host_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q,
                           const float *dq, int64_t B, const abrb_rbd_out *out);

/* ---------------------------------------------------------------------------------------------------
 * Operational-space controller.  abrb_osc_params mirrors the constructor of
 * abr_control.controllers.OSC (controllers/osc.py:53-118) plus its secondary ("null space") controllers:
 *   ABRB_NULL_DAMPING        controllers/damping.py:21-32          M (-kv dq)
 *   ABRB_NULL_RESTING        controllers/resting_config.py:25-42 + controllers/joint.py:104-131
 *   ABRB_NULL_AVOID          controllers/avoid_obstacles.py:38-120
 * abrb_osc_generate_* evaluates OSC.generate (controllers/osc.py:217-320) for B states.
 * ------------------------------------------------------------------------------------------------- */
enum { ABRB_NULL_DAMPING = 1, ABRB_NULL_RESTING = 2, ABRB_NULL_AVOID = 3, ABRB_NULL_JOINT_LIMITS = 4 };

typedef struct abrb_null_params {
  int32_t kind;
  int32_t n_obstacles;                            /* AVOID */
  double kp, kv;                                  /* DAMPING: kv; RESTING: kp, kv (Joint: kv default sqrt(kp)) */
  double rest_angles[ABRB_MAX_JOINTS];            /* RESTING */
  int32_t rest_mask[ABRB_MAX_JOINTS];             /* RESTING: 0 where the reference has None */
  int32_t _pad;
  double threshold, gain, maximum;                /* AVOID (avoid_obstacles.py:25-36) */
  double obstacles[ABRB_MAX_OBSTACLES][4];        /* AVOID: x, y, z, radius */
  /* JOINT_LIMITS (avoid_joint_limits.py:36-86): the controller's attributes AFTER its constructor, i.e. limits
   * shifted by -pi and swapped where cross_zero is set; NaN = no limit on that side; max_torque default 1 */
  double limit_min[ABRB_MAX_JOINTS], limit_max[ABRB_MAX_JOINTS], limit_torque[ABRB_MAX_JOINTS];
  int32_t limit_cross_zero[ABRB_MAX_JOINTS], limit_gradient[ABRB_MAX_JOINTS];
} abrb_null_params;

typedef struct abrb_osc_params {
  double kp, ko, kv, ki;                          /* resolved gains: caller applies the ko/kv defaults (osc.py:71-74) */
  double vmax[2];                                 /* used if use_vmax */
  double mx_threshold;                            /* `_Mx(threshold=1e-3)`, osc.py:120 */
  int32_t use_vmax;
  int32_t ctrlr_dof[6];
  int32_t use_g, use_C;
  int32_t orientation_algorithm;                  /* 0 or 1, else ABRB_EUNSUP */
  int32_t n_null;
  int32_t _pad;
  abrb_null_params null[ABRB_MAX_NULL];
} abrb_osc_params;

typedef struct abrb_osc abrb_osc;

int abrb_osc_create(const abrb_model *m, const abrb_osc_params *p, abrb_osc **out);
int abrb_osc_destroy(abrb_osc *c);

/* Execution options of one controller (no effect on results).  Names:
 *   "host_chunk_states"  states per pipeline chunk of the *_host entry points; 0 = automatic (default: the blocking
 *                        calls split batches of 49 152 states and more into two chunks, four above 196 608; the
 *                        asynchronous calls, which overlap whole calls on the two slots, keep one chunk up to 196 608
 *                        states; the environment variable ABRB_HOST_CHUNK sets another default).
 *   "host_upload_streams" copy streams per chunk of the *_host entry points: 1 (q, dq, target one after the other), 2
 *                        (default: dq beside q) or 3 (per-state targets on a stream of their own as well); default from
 *                        ABRB_HOST_STREAMS.  Which is fastest depends on the host: one pinned host->device stream
 *                        can reach very different rates on different machines.
 * Returns ABRB_EINVAL for an unknown name.  Not thread safe against concurrent generate calls on the same handle. */
int abrb_osc_set_option(abrb_osc *c, const char *name, double value);

/* OSC.generate(q, dq, target, target_velocity=None, ref_frame="EE", xyz_offset=None) for B states.
 *   target           (B,6) if target_stride == 6, or one (6,) row broadcast to all states if target_stride == 0
 *   target_velocity  NULL (the reference's `np.all(target_velocity == 0)` joint-space damping branch,
 *                    osc.py:275-278) or (B,6)/(6,) per tv_stride (task-space branch, osc.py:279-282)
 *   u                (B,n) out;   training_signal (B,n) out or NULL (osc.py:297)
 *   integrated_error (B,6) in/out: the reference's per-controller `self.integrated_error` (osc.py:81-82), one row per
 *                    state, updated as osc.py:262-264 (`integrated_error += u_task; u_task += ki * integrated_error`).
 *                    Must be given if and only if the controller was created with ki != 0 (else ABRB_EINVAL); the
 *                    caller owns it and zeroes it to reset the integrator.
 *   frame_id/x_off   ref_frame and xyz_offset (x_off: 3 host doubles or NULL) */
int abrb_osc_generate_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q,
                          const double *dq, const double *target, int target_stride,
                          const double *target_velocity, int tv_stride, double *u,
                          double *training_signal, double *integrated_error, int64_t B, void *stream);
int abrb_osc_generate_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q,
                          const float *dq, const float *target, int target_stride,
                          const float *target_velocity, int tv_stride, float *u,
                          float *training_signal, float *integrated_error, int64_t B, void *stream);
/* HOST-pointer variants (H2D + kernel + D2H + sync inside) */
int abrb_osc_generate_host_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q,
                               const double *dq, const double *target, int target_stride,
                               const double *target_velocity, int tv_stride, double *u,
                               double *training_signal, double *integrated_error, int64_t B);
int abrb_osc_generate_host_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q,
                               const float *dq, const float *target, int target_stride,
                               const float *target_velocity, int tv_stride, float *u,
                               float *training_signal, float *integrated_error, int64_t B);
/* Asynchronous HOST-pointer variants for control loops that evaluate batch after batch: the call enqueues the H2D
 * copies, the kernel and the D2H copies of one batch on pipeline slot `slot` (0 or 1) of the calling thread and
 * returns; abrb_osc_host_wait(c, slot) blocks until that batch's outputs are in the caller's buffers.  With the two
 * slots used alternately, batch k+1's H2D runs under batch k's kernel and D2H (PCIe is full duplex), so a stream of
 * calls costs max(H2D, kernel, D2H) per batch instead of their sum.  The host buffers (page-locked for real
 * asynchrony) must stay valid and untouched until the wait; enqueueing on a slot first waits for its previous batch.
 * The synchronous variants above are slot 0 + wait. */
int abrb_osc_generate_host_async_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q,
                                     const double *dq, const double *target, int target_stride,
                                     const double *target_velocity, int tv_stride, double *u,
                                     double *training_signal, double *integrated_error, int64_t B, int slot);
int abrb_osc_generate_host_async_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q,
                                     const float *dq, const float *target, int target_stride,
                                     const float *target_velocity, int tv_stride, float *u,
                                     float *training_signal, float *integrated_error, int64_t B, int slot);
int abrb_osc_host_wait(const abrb_osc *c, int slot);

/* ---------------------------------------------------------------------------------------------------
 * Fused all-gather of the control outputs across the GPUs of one box (BASELINE config 5, SURVEY.md S8e): one
 * process per GPU, every rank evaluates its own row block, and the OSC kernel's epilogue stores each finished tile of
 * `u` straight into the gathered (B_total, n) array of EVERY rank through NVLink peer memory (buffers mapped with CUDA
 * IPC) — the exchange overlaps the arithmetic instead of following it as a separate NCCL collective.
 *   abrb_gather_create   allocates this rank's region: n_buffers gathered arrays of bytes_per_buffer each (use two and
 *                        alternate them call by call: a fast rank may already write call k+1 while a slow one still
 *                        reads call k) plus the completion flags
 *   abrb_gather_export / abrb_gather_import   exchange the 64-byte CUDA IPC handles (any transport: MPI,
 *                        torch.distributed.all_gather_object, a file); every rank imports every other rank once
 *   abrb_osc_generate_gather_*   abrb_osc_generate_* whose rows additionally land at row `row0` of buffer
 *                        `buffer_index` on every rank (`u` may be NULL if only the gathered copy is wanted); all ranks
 *                        must make the same sequence of gather calls
 *   abrb_gather_wait     enqueues, on `stream`, a wait until every rank's rows of the latest gather call have arrived
 *                        in this rank's buffer (device-side spin on the flags; gives up after ~3 s and sets the status)
 *   abrb_gather_buffer   device pointer of this rank's gathered array `buffer_index`
 *   abrb_gather_status   0, or 1 if a wait ever timed out (call after synchronising the stream)
 * ------------------------------------------------------------------------------------------------- */
typedef struct abrb_gather abrb_gather;
int abrb_gather_create(int rank, int world, int64_t bytes_per_buffer, int n_buffers, abrb_gather **out);
int abrb_gather_destroy(abrb_gather *g);
int abrb_gather_export(const abrb_gather *g, unsigned char handle[64]);
int abrb_gather_import(abrb_gather *g, int peer_rank, const unsigned char handle[64]);
void *abrb_gather_buffer(const abrb_gather *g, int buffer_index);
int abrb_gather_wait(abrb_gather *g, void *stream);
int abrb_gather_status(const abrb_gather *g);
int abrb_osc_generate_gather_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q,
                                 const double *dq, const double *target, int target_stride,
                                 const double *target_velocity, int tv_stride, double *u, double *training_signal,
                                 double *integrated_error, int64_t B, abrb_gather *g, int buffer_index, int64_t row0,
                                 void *stream);
int abrb_osc_generate_gather_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q,
                                 const float *dq, const float *target, int target_stride,
                                 const float *target_velocity, int tv_stride, float *u, float *training_signal,
                                 float *integrated_error, int64_t B, abrb_gather *g, int buffer_index, int64_t row0,
                                 void *stream);

/* Standalone secondary controller: Damping / RestingConfig / AvoidObstacles / AvoidJointLimits
 * `.generate(q, dq)` -> (B,n). */
int abrb_null_generate_f64(const abrb_model *m, const abrb_null_params *p, const double *q,
                           const double *dq, double *u, int64_t B, void *stream);
int abrb_null_generate_f32(const abrb_model *m, const abrb_null_params *p, const float *q,
                           const float *dq, float *u, int64_t B, void *stream);

/* Joint-space PD controller  Joint.generate(q, dq, target, target_velocity=None)
 * (controllers/joint.py:104-131):  u = M (kp q_tilde + kv (target_velocity - dq)) [- g],
 * q_tilde = ((target - q + pi) mod 2 pi) - pi  (joint.py:42-46; the ball-joint/quaternion branch is MuJoCo-only).
 *   target (B,n) if target_stride == n, one (n,) row if 0;  target_velocity NULL or per tv_stride. */
int abrb_joint_generate_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, const double *q,
                            const double *dq, const double *target, int target_stride,
                            const double *target_velocity, int tv_stride, double *u, int64_t B, void *stream);
int abrb_joint_generate_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, const float *q,
                            const float *dq, const float *target, int target_stride,
                            const float *target_velocity, int tv_stride, float *u, int64_t B, void *stream);

/* Gravity compensation  Floating.generate(q, dq)  (controllers/floating.py:27-71):
 *   joint space:  u = -g;   task space:  u = J^T (-(M^-1 J^T Mx)^T g) with J = J("EE")[:3] and the reference's
 *   inv / pinv(rcond=1e-4) switch at |det| > 1e-3;   dynamic: u -= M dq.   dq may be NULL unless dynamic. */
int abrb_floating_generate_f64(const abrb_model *m, int task_space, int dynamic, const double *q, const double *dq,
                               double *u, int64_t B, void *stream);
int abrb_floating_generate_f32(const abrb_model *m, int task_space, int dynamic, const float *q, const float *dq,
                               float *u, int64_t B, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * Closed-loop rollout (SURVEY.md S8d config 4, S8f#1): `steps` iterations of
 *     u = OSC.generate(q, dq, target);  ddq = M^-1 (u + g - C dq);  dq += ddq dt;  q += dq dt
 * (semi-implicit Euler as the reference's in-repo plant, arms/twojoint/arm_sim.py:131-132; the reference
 * has no plant for UR5/Jaco2, this one uses the same M, g, C the controller uses).
 *   q, dq   (B,n) in/out (final state);  target (B,6) or (6,) per target_stride
 *   q_traj / dq_traj / u_traj: NULL or (steps, B, n) outputs
 *   integrated_error: (B,6) in/out, given if and only if ki != 0 (as for abrb_osc_generate_*)
 * ------------------------------------------------------------------------------------------------- */
int abrb_osc_rollout_f64(const abrb_osc *c, int frame_id, const double *x_off, double *q, double *dq,
                         const double *target, int target_stride, int steps, double dt,
                         double *q_traj, double *dq_traj, double *u_traj, double *integrated_error, int64_t B,
                         void *stream);
int abrb_osc_rollout_f32(const abrb_osc *c, int frame_id, const double *x_off, float *q, float *dq,
                         const float *target, int target_stride, int steps, double dt,
                         float *q_traj, float *dq_traj, float *u_traj, float *integrated_error, int64_t B,
                         void *stream);

/* ---------------------------------------------------------------------------------------------------
 * Path-following rollout (MPC over a reference trajectory): the closed loop of abrb_osc_rollout_*, but step t
 * drives towards the path's row p_t (x, y, z, Euler a, b, g, as generate's target) with target velocity v_t,
 * and the control point's track and one tracking cost per trajectory are recorded.  For t = 0 .. steps-1:
 *     x_t      = position of the control point (frame_id + x_off) at q_t
 *     u_t      = OSC.generate(q_t, dq_t, target = p_t, target_velocity = v_t)
 *                (v_t all zero or path_velocity NULL: the -kv M dq law, as generate)
 *     ddq_t    = M(q_t)^-1 (u_t + g(q_t) - C(q_t, dq_t) dq_t)
 *     dq_{t+1} = dq_t + ddq_t dt;   q_{t+1} = q_t + dq_{t+1} dt          (semi-implicit Euler, as the rollout)
 *     cost    += |x_t - p_t[0:3]|^2 + effort_weight |u_t|^2              (in order of t, in the call's precision;
 *                                                                          position rows even when not controlled)
 * x_traj[t] and u_traj[t] belong to the state BEFORE step t; q_traj[t] and dq_traj[t] hold the state AFTER it.
 *   q, dq          (B,n) in/out (final state)
 *   path           path_stride 6: (steps, B, 6), element (t, b, c) at path[(t*B + b)*6 + c] (one path per trajectory);
 *                  path_stride 0: (steps, 6), element (t, c) at path[t*6 + c] (one path shared by all)
 *   path_velocity  NULL or laid out like path per pv_stride (0 or 6)
 *   q_traj / dq_traj / u_traj: NULL or (steps, B, n);   x_traj: NULL or (steps, B, 3);   cost: NULL or (B,)
 *   effort_weight  finite, >= 0 (double for both precisions, as dt)
 *   integrated_error: (B,6) in/out, given if and only if ki != 0; the rollout starts from it and leaves it updated
 * steps == 0 leaves q, dq unchanged and writes cost = 0; B == 0 does nothing.  Arguments are checked before any
 * device work: ABRB_EINVAL (NULL controller, q, dq, or path when steps > 0; strides other than 0 or 6; negative
 * steps or B; effort_weight negative or not finite; integrated_error / ki mismatch; misaligned pointers),
 * ABRB_EFRAME (bad frame id).
 * ------------------------------------------------------------------------------------------------- */
int abrb_osc_rollout_path_f64(const abrb_osc *c, int frame_id, const double *x_off, double *q, double *dq,
                              const double *path, int path_stride, const double *path_velocity, int pv_stride,
                              int steps, double dt, double effort_weight,
                              double *q_traj, double *dq_traj, double *u_traj, double *x_traj, double *cost,
                              double *integrated_error, int64_t B, void *stream);
int abrb_osc_rollout_path_f32(const abrb_osc *c, int frame_id, const double *x_off, float *q, float *dq,
                              const float *path, int path_stride, const float *path_velocity, int pv_stride,
                              int steps, double dt, double effort_weight,
                              float *q_traj, float *dq_traj, float *u_traj, float *x_traj, float *cost,
                              float *integrated_error, int64_t B, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * The rollouts' plant on its own, for torques from anywhere (sampling-based MPC in torque space, other
 * controllers, replay of a recorded u_traj, feedforward torques of a planned joint trajectory).  It is the plant
 * of abrb_osc_rollout_* (semi-implicit Euler as arms/twojoint/arm_sim.py:131-132), with g the generalized gravity
 * force the controllers subtract (base_config.py:417-468) and C dq the rollout's Coriolis product:
 *     forward dynamics   ddq = M(q)^-1 (u + g(q) - C(q, dq) dq)
 *     inverse dynamics   u   = M(q) ddq + C(q, dq) dq - g(q)
 *   q, dq, u, ddq (B,n).  B == 0 does nothing.  ABRB_EINVAL: NULL model or array, B < 0, misaligned pointers.
 * ------------------------------------------------------------------------------------------------- */
int abrb_forward_dynamics_f64(const abrb_model *m, const double *q, const double *dq, const double *u,
                              double *ddq, int64_t B, void *stream);
int abrb_forward_dynamics_f32(const abrb_model *m, const float *q, const float *dq, const float *u,
                              float *ddq, int64_t B, void *stream);
int abrb_inverse_dynamics_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq,
                              double *u, int64_t B, void *stream);
int abrb_inverse_dynamics_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq,
                              float *u, int64_t B, void *stream);

/* Inverse-dynamics regressor.  Inverse dynamics is linear in the diagonal link inertias:
 *     u = M(q) ddq + C(q, dq) dq - g(q) = Y(q, dq, ddq) theta,   theta[6 (l-1) + c] = link_inertia[l][c]
 * for links l = 1 .. n and c = 0..5 (m_x, m_y, m_z, I_xx, I_yy, I_zz); link 0 never enters.  Writes Y^T per state:
 *   q, dq, ddq     (B,n)
 *   Yt             (B, 6n, n), element (b, p, a) at Yt[(b*6n + p)*n + a] = d u_a / d theta_p of state b, so the 6n
 *                  values of link l (rows 6(l-1) .. 6l-1) are contiguous in each state's record
 * With theta the model's own constants, sum_p Yt[b, p, :] theta[p] is abrb_inverse_dynamics_* of the same state (to
 * rounding).  The model's gravity is used.  B == 0 does nothing.  Arguments are checked before any device work:
 * ABRB_EINVAL (NULL model or array, B < 0, misaligned pointers).
 * ------------------------------------------------------------------------------------------------- */
int abrb_inverse_dynamics_regressor_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq,
                                        double *Yt, int64_t B, void *stream);
int abrb_inverse_dynamics_regressor_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq,
                                        float *Yt, int64_t B, void *stream);

/* Open-loop plant rollout under a given torque sequence u_t.  For t = 0 .. steps-1:
 *     tau_t    = u_t                       (compensate_gravity == 0)
 *     tau_t    = u_t - g(q_t)              (compensate_gravity != 0: u_t is the residual torque MPPI samples around)
 *     x_t      = position of the control point (frame_id + x_off) at q_t
 *     ddq_t    = M(q_t)^-1 (tau_t + g(q_t) - C(q_t, dq_t) dq_t)
 *     dq_{t+1} = dq_t + ddq_t dt;   q_{t+1} = q_t + dq_{t+1} dt
 *     cost    += |x_t - p_t[0:3]|^2 (with a path only) + effort_weight |tau_t|^2   (in order of t, in the call's
 *                                                                                  precision)
 * The records follow abrb_osc_rollout_path_*: x_traj[t] and u_traj[t] (the applied tau_t) belong to the state
 * BEFORE step t, q_traj[t] and dq_traj[t] hold the state AFTER it; the cost is the same sum.  So the u_traj of a
 * closed-loop path rollout, fed back here with the same path and effort_weight, gives back that rollout's track and
 * cost, and closed-loop and open-loop candidates are scored alike.
 *   q, dq          (B,n) in/out (final state)
 *   u              u_stride n: (steps, B, n), element (t, b, k) at u[(t*B + b)*n + k] (one sequence per trajectory);
 *                  u_stride 0: (steps, n), element (t, k) at u[t*n + k] (one sequence shared by all)
 *   path           NULL or laid out as in abrb_osc_rollout_path_* per path_stride (6 or 0); columns 0-2 are used
 *   q_traj / dq_traj / u_traj: NULL or (steps, B, n);   x_traj: NULL or (steps, B, 3);   cost: NULL or (B,)
 *   effort_weight  finite, >= 0 (double for both precisions, as dt)
 * steps == 0 leaves q, dq unchanged and writes cost = 0; B == 0 does nothing.  Arguments are checked before any
 * device work: ABRB_EINVAL (NULL model, q, dq, or u when steps > 0; u_stride other than 0 or n; path_stride other
 * than 0 or 6; negative steps or B; effort_weight negative or not finite; misaligned pointers), ABRB_EFRAME (bad
 * frame id).
 * ------------------------------------------------------------------------------------------------- */
int abrb_plant_rollout_f64(const abrb_model *m, int frame_id, const double *x_off, double *q, double *dq,
                           const double *u, int u_stride, int compensate_gravity,
                           const double *path, int path_stride, int steps, double dt, double effort_weight,
                           double *q_traj, double *dq_traj, double *u_traj, double *x_traj, double *cost,
                           int64_t B, void *stream);
int abrb_plant_rollout_f32(const abrb_model *m, int frame_id, const double *x_off, float *q, float *dq,
                           const float *u, int u_stride, int compensate_gravity,
                           const float *path, int path_stride, int steps, double dt, double effort_weight,
                           float *q_traj, float *dq_traj, float *u_traj, float *x_traj, float *cost,
                           int64_t B, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * Derivatives of the plant (forward-mode dual numbers through the same per-state code, DESIGN.md S3.6).
 * Every derivative is (B, n, n) row-major, element [b, i, j] = d out_i / d in_j:
 *   forward:  d_q = d ddq / d q,  d_dq = d ddq / d dq,  d_u = d ddq / d u = M^-1   (d_u may be NULL)
 *   inverse:  d_q = d u / d q,    d_dq = d u / d dq,    d_ddq = d u / d ddq = M    (d_ddq may be NULL)
 * B == 0 does nothing.  ABRB_EINVAL: NULL model or required array, B < 0, misaligned pointers.
 * ------------------------------------------------------------------------------------------------- */
int abrb_forward_dynamics_derivatives_f64(const abrb_model *m, const double *q, const double *dq, const double *u,
                                          double *d_q, double *d_dq, double *d_u, int64_t B, void *stream);
int abrb_forward_dynamics_derivatives_f32(const abrb_model *m, const float *q, const float *dq, const float *u,
                                          float *d_q, float *d_dq, float *d_u, int64_t B, void *stream);
int abrb_inverse_dynamics_derivatives_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq,
                                          double *d_q, double *d_dq, double *d_ddq, int64_t B, void *stream);
int abrb_inverse_dynamics_derivatives_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq,
                                          float *d_q, float *d_dq, float *d_ddq, int64_t B, void *stream);

/* Vector-Jacobian product of abrb_plant_rollout_*: given the rollout's arguments (q0, dq0: the START state), the
 * states it recorded (q_traj, dq_traj: (steps, B, n), required when steps > 0) and cotangents of its outputs, each
 * NULL (zero) or
 *     g_cost (B),  g_q, g_dq (B,n) of the final state,  g_q_traj, g_dq_traj, g_u_traj (steps, B, n),  g_x_traj
 *     (steps, B, 3)
 * writes the cotangents gu (steps, B, n) of the torques — per trajectory also for a shared (u_stride 0) sequence,
 * whose gradient is their sum over B — and gq0, gdq0 (B,n) of the start state.  Backward recursion over
 * t = S-1 .. 0 with mu_S = (g_q, g_dq), x_t = (q_t, dq_t) the state before step t and Phi_t the step:
 *     mu_{t+1} += (g_q_traj[t], g_dq_traj[t])
 *     lambda_t  = g_cost dc_t/dx_t + g_x_traj[t] dx_t/dx_t + g_u_traj[t] dtau_t/dx_t + (dPhi_t/dx_t)^T mu_{t+1}
 *     gu[t]     = g_cost dc_t/du_t + g_u_traj[t] dtau_t/du_t + (dPhi_t/du_t)^T mu_{t+1};     mu_t = lambda_t
 * and (gq0, gdq0) = lambda_0 (= (g_q, g_dq) for steps == 0).  The path, dt and effort_weight are constants.
 * Argument errors as abrb_plant_rollout_*, plus NULL q0, dq0, gq0, gdq0, and (steps > 0) NULL u, q_traj, dq_traj,
 * gu: ABRB_EINVAL.
 * ------------------------------------------------------------------------------------------------- */
int abrb_plant_rollout_vjp_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q0,
                               const double *dq0, const double *u, int u_stride, int compensate_gravity,
                               const double *path, int path_stride, int steps, double dt, double effort_weight,
                               const double *q_traj, const double *dq_traj, const double *g_cost, const double *g_q,
                               const double *g_dq, const double *g_q_traj, const double *g_dq_traj,
                               const double *g_u_traj, const double *g_x_traj, double *gu, double *gq0, double *gdq0,
                               int64_t B, void *stream);
int abrb_plant_rollout_vjp_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q0,
                               const float *dq0, const float *u, int u_stride, int compensate_gravity,
                               const float *path, int path_stride, int steps, double dt, double effort_weight,
                               const float *q_traj, const float *dq_traj, const float *g_cost, const float *g_q,
                               const float *g_dq, const float *g_q_traj, const float *g_dq_traj,
                               const float *g_u_traj, const float *g_x_traj, float *gu, float *gq0, float *gdq0,
                               int64_t B, void *stream);

/* Gradient of abrb_plant_rollout_* with respect to the link inertias theta = link_inertia[1:] flattened (theta[6 (l-1)
 * + c], as abrb_inverse_dynamics_regressor_*).  Given the rollout's start state, torques and recorded states (q_traj,
 * dq_traj: (steps, B, n)), the torque cotangents gu (steps, B, n) that abrb_plant_rollout_vjp_* wrote for the same
 * output cotangents, and the cotangents g_cost (B) and g_u_traj (steps, B, n) of the cost and of the recorded torques
 * (each NULL: zero), writes
 *     g_theta (B, 6n) = sum_t [ -Y(q_t, dq_t, ddq_t)^T w_t + c_g Y(q_t, 0, 0)^T gu_t ],
 *     w_t = gu_t - 2 effort_weight g_cost tau_t - g_u_traj[t]
 * per trajectory (the gradient of the shared model is the sum over B).  (q_t, dq_t) is the state before step t, tau_t
 * its applied torque, ddq_t = M^-1 (tau_t + g - C dq_t) recomputed from them, c_g = 1 with compensate_gravity and 0
 * without.  The frame, offset and path do not depend on theta; dt enters through gu.  steps == 0 writes zeros, B == 0
 * does nothing.  No atomics: rows are bit-identical between runs and under a permutation of the trajectories.
 * Argument errors (before any device work) as abrb_plant_rollout_vjp_*: ABRB_EINVAL for a NULL model, q0, dq0 or
 * g_theta, (steps > 0) a NULL u, q_traj, dq_traj or gu, B < 0, steps < 0, u_stride not 0 or n, a negative or
 * non-finite effort_weight, misaligned pointers.
 * ------------------------------------------------------------------------------------------------- */
int abrb_plant_rollout_theta_vjp_f64(const abrb_model *m, const double *q0, const double *dq0, const double *u,
                                     int u_stride, int compensate_gravity, int steps, double effort_weight,
                                     const double *q_traj, const double *dq_traj, const double *gu,
                                     const double *g_cost, const double *g_u_traj, double *g_theta, int64_t B,
                                     void *stream);
int abrb_plant_rollout_theta_vjp_f32(const abrb_model *m, const float *q0, const float *dq0, const float *u,
                                     int u_stride, int compensate_gravity, int steps, double effort_weight,
                                     const float *q_traj, const float *dq_traj, const float *gu, const float *g_cost,
                                     const float *g_u_traj, float *g_theta, int64_t B, void *stream);

/* Vector-Jacobian product of abrb_joint_rollout_path_*: given the rollout's arguments (q0, dq0: the START state), the
 * states it recorded (q_traj, dq_traj: (steps, B, n), required when steps > 0) and cotangents of its outputs, each
 * NULL (zero) or as in abrb_plant_rollout_vjp_* (g_u_traj: of the recorded Joint torques u), writes
 *     g_path, g_path_velocity (steps, B, n): the cotangents of the path and path velocity rows — per trajectory also
 *         for a shared (stride 0) path, whose gradient is their sum over B; NULL: not wanted
 *     g_gains (B, 2): [d/dkp, d/dkv] per trajectory (the gradient of the scalar gains is their sum over B); NULL: not
 *         wanted
 *     gq0, gdq0 (B, n): the cotangents of the start state.
 * Backward recursion over t = S-1 .. 0 with mu_S = (g_q, g_dq), x_t = (q_t, dq_t) the state before step t, Phi_t the
 * closed-loop step, theta_t = (path[t], path_velocity[t]) and gamma = (kp, kv):
 *     mu_{t+1} += (g_q_traj[t], g_dq_traj[t])
 *     lambda_t  = g_cost dc_t/dx_t + g_x_traj[t] dx^_t/dx_t + g_u_traj[t] du_t/dx_t + (dPhi_t/dx_t)^T mu_{t+1}
 *     g_theta[t] = g_cost dc_t/dtheta_t + g_u_traj[t] du_t/dtheta_t + (dPhi_t/dtheta_t)^T mu_{t+1}
 *     g_gamma  += g_cost dc_t/dgamma + g_u_traj[t] du_t/dgamma + (dPhi_t/dgamma)^T mu_{t+1};     mu_t = lambda_t
 * and (gq0, gdq0) = lambda_0 (= (g_q, g_dq) and zero gains for steps == 0).  The wrap of path - q passes the tangent
 * through unchanged; dt, effort_weight, account_for_gravity, the frame and x_off are constants.  Argument errors as
 * abrb_joint_rollout_path_*, plus NULL q0, dq0, gq0, gdq0, (steps > 0) NULL path, q_traj, dq_traj, and a g_path_velocity
 * without a path_velocity: ABRB_EINVAL.
 * ------------------------------------------------------------------------------------------------- */
int abrb_joint_rollout_path_vjp_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                    const double *x_off, const double *q0, const double *dq0, const double *path,
                                    int path_stride, const double *path_velocity, int pv_stride, int steps, double dt,
                                    double effort_weight, const double *q_traj, const double *dq_traj,
                                    const double *g_cost, const double *g_q, const double *g_dq,
                                    const double *g_q_traj, const double *g_dq_traj, const double *g_u_traj,
                                    const double *g_x_traj, double *g_path, double *g_path_velocity, double *g_gains,
                                    double *gq0, double *gdq0, int64_t B, void *stream);
int abrb_joint_rollout_path_vjp_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                    const double *x_off, const float *q0, const float *dq0, const float *path,
                                    int path_stride, const float *path_velocity, int pv_stride, int steps, double dt,
                                    double effort_weight, const float *q_traj, const float *dq_traj,
                                    const float *g_cost, const float *g_q, const float *g_dq, const float *g_q_traj,
                                    const float *g_dq_traj, const float *g_u_traj, const float *g_x_traj,
                                    float *g_path, float *g_path_velocity, float *g_gains, float *gq0, float *gdq0,
                                    int64_t B, void *stream);

/* Kernel launch counter for this process (every launch of a libabrb kernel increments it). */
int64_t abrb_launch_count(void);

/* Sliding-mode controller  Sliding.generate(q, dq, target, target_velocity=0, target_acc=0, ref_frame="EE",
 * offset=None)  (controllers/sliding.py:34-99):
 *   cartesian != 0:  J = J(frame, x_off)[:3], dq_ref = pinv(J)(tv + lamb (target - Tx)),
 *                    ddq_ref = pinv(J)(ta + lamb (tv - J dq) - dJ[:3] dq_ref);   target/tv/ta rows have 3 values
 *   cartesian == 0:  dq_ref = tv - lamb (q - target), ddq_ref = ta - lamb (dq - tv);   rows have n values
 *   s = dq - dq_ref,  u = M ddq_ref + C dq_ref + g - kd s.
 * target: one row per state (stride = row width) or one broadcast row (stride 0); target_velocity / target_acc
 * likewise or NULL (zero).  s (B,n) receives the reference's `self.s` (the adaptation signal) or may be NULL. */
int abrb_sliding_generate_f64(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                              const double *x_off, const double *q, const double *dq, const double *target,
                              int target_stride, const double *target_velocity, int tv_stride,
                              const double *target_acc, int ta_stride, double *u, double *s, int64_t B,
                              void *stream);
int abrb_sliding_generate_f32(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                              const double *x_off, const float *q, const float *dq, const float *target,
                              int target_stride, const float *target_velocity, int tv_stride,
                              const float *target_acc, int ta_stride, float *u, float *s, int64_t B, void *stream);

/* Iterative inverse-kinematics path  InverseKinematics(robot_config, max_dx, max_dr, max_dq).generate_path(position,
 * target_position, n_timesteps, dt, method)  (controllers/path_planners/inverse_kinematics.py:28-166), one path per
 * state: n_timesteps resolved-motion steps towards target (x, y, z, Euler a, b, g) at frame "EE", the task-space
 * step clipped to max_dx dt / max_dr dt and the joint step to max_dq dt.  method 1: pinv(J); 2: damped least
 * squares; 3: position first, orientation in its null space (the reference's default).
 *   position (B,n);  target (B,6) if target_stride == 6, one (6,) row if 0
 *   position_path, velocity_path: (n_timesteps, B, n) out — row t holds q_t and the step dq_t taken from it */
int abrb_ik_path_f64(const abrb_model *m, double max_dx, double max_dr, double max_dq, int method, double dt,
                     int n_timesteps, const double *position, const double *target, int target_stride,
                     double *position_path, double *velocity_path, int64_t B, void *stream);
int abrb_ik_path_f32(const abrb_model *m, double max_dx, double max_dr, double max_dq, int method, double dt,
                     int n_timesteps, const float *position, const float *target, int target_stride,
                     float *position_path, float *velocity_path, int64_t B, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * Closed-loop rollouts of Joint and Sliding along a path, the counterpart of abrb_osc_rollout_path_* for the other
 * trajectory-tracking controllers.  For t = 0 .. steps-1, from the state (q_t, dq_t) before the step:
 *     u_t      = Joint.generate(q_t, dq_t, path_t, path_velocity_t)      (as abrb_joint_generate_*)
 *     u_t      = Sliding.generate(q_t, dq_t, path_t, path_velocity_t, path_acc_t, frame_id, x_off)
 *                                                                          (as abrb_sliding_generate_*)
 *     x_t      = position of the control point (frame_id + x_off) at q_t
 *     ddq_t    = M(q_t)^-1 (u_t + g(q_t) - C(q_t, dq_t) dq_t)
 *     dq_{t+1} = dq_t + ddq_t dt;   q_{t+1} = q_t + dq_{t+1} dt
 *     cost    += e_t + effort_weight |u_t|^2,   e_t = |wrap_pm_pi(path_t - q_t)|^2   (Joint)
 *                                               e_t = |x_t - path_t|^2             (Sliding, cartesian != 0)
 *                                               e_t = |q_t - path_t|^2             (Sliding, joint mode; not wrapped)
 * The plant is that of abrb_plant_rollout_*, so u_traj replayed there (no path, same effort_weight) gives back q, dq
 * and x.  Sliding keeps the reference's +g (sliding.py:97): with gravity the closed loop runs against a 2 g bias.
 * Records as abrb_plant_rollout_*: x_traj[t] and u_traj[t] belong to the state BEFORE step t, q_traj[t] and
 * dq_traj[t] to the state AFTER it.  In joint-mode Sliding, frame_id and x_off only choose the recorded x.
 *   q, dq          (B,n) in/out (final state)
 *   path, path_velocity, path_acc: rows of width w = 3 (cartesian Sliding) or n; stride w: (steps, B, w), element
 *                  (t, b, k) at [(t*B + b)*w + k]; stride 0: one (steps, w) sequence for every trajectory.
 *                  path_velocity and path_acc may be NULL (zero).
 *   q_traj / dq_traj / u_traj: NULL or (steps, B, n);   x_traj: NULL or (steps, B, 3);   cost: NULL or (B,)
 *   effort_weight  finite, >= 0 (double for both precisions, as dt, the gains and x_off)
 * steps == 0 leaves q, dq unchanged and writes cost = 0; B == 0 does nothing.  Arguments are checked before any
 * device work: ABRB_EINVAL (NULL model, q, dq, or path when steps > 0; a stride other than 0 or w; negative steps or
 * B; effort_weight negative or not finite; misaligned pointers), ABRB_EFRAME (bad frame id).
 * ------------------------------------------------------------------------------------------------- */
int abrb_joint_rollout_path_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                const double *x_off, double *q, double *dq, const double *path, int path_stride,
                                const double *path_velocity, int pv_stride, int steps, double dt,
                                double effort_weight, double *q_traj, double *dq_traj, double *u_traj,
                                double *x_traj, double *cost, int64_t B, void *stream);
int abrb_joint_rollout_path_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                const double *x_off, float *q, float *dq, const float *path, int path_stride,
                                const float *path_velocity, int pv_stride, int steps, double dt, double effort_weight,
                                float *q_traj, float *dq_traj, float *u_traj, float *x_traj, float *cost, int64_t B,
                                void *stream);
int abrb_sliding_rollout_path_f64(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                                  const double *x_off, double *q, double *dq, const double *path, int path_stride,
                                  const double *path_velocity, int pv_stride, const double *path_acc, int pa_stride,
                                  int steps, double dt, double effort_weight, double *q_traj, double *dq_traj,
                                  double *u_traj, double *x_traj, double *cost, int64_t B, void *stream);
int abrb_sliding_rollout_path_f32(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                                  const double *x_off, float *q, float *dq, const float *path, int path_stride,
                                  const float *path_velocity, int pv_stride, const float *path_acc, int pa_stride,
                                  int steps, double dt, double effort_weight, float *q_traj, float *dq_traj,
                                  float *u_traj, float *x_traj, float *cost, int64_t B, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * Batched path planner  PathPlanner(pos_profile, vel_profile, axes).generate_path(start, target, max_velocity,
 * start_orientation, target_orientation, start_velocity, target_velocity)  (controllers/path_planners/path_planner.py),
 * one path per row.  The position profile enters as its table  table[i] = pos_profile.step(i / (n_points - 1)),
 * (n_points, 3) row-major fp64 on the device; the velocity profile by kind and parameters.  All planning arithmetic is
 * fp64 in both entry points of phase 2; only the stored rows are float in abrb_path_fill_f32.
 *
 * Phase 1, abrb_path_plan: per row, the warped curve's length and the reference's max_v search (starting from
 * max_velocity, stepping down by 0.1).  lengths[b] is the row's number of steps S_b, or a negative ABRB_PATH_* reason
 * when the reference cannot plan it; plan[b] is the record phase 2 needs.
 * Phase 2, abrb_path_fill_*: path (s_max, B, w), w = 12 with orientations (x, dx, Euler angles, their gradient) and 6
 * without; rows S_b .. s_max-1 repeat row S_b - 1.  Rows with lengths[b] < 2 are filled with NaN.
 * Inputs of both phases: start, target (B,3); max_velocity, start_velocity, target_velocity (B,); orientations (B,3)
 * Euler angles in the order params->axes.  All pointers are device pointers. */
#define ABRB_PATH_MAX_POINTS 4096 /* n_points bound: phase 2 keeps 32 bytes per point in shared memory */
enum { ABRB_VEL_GAUSSIAN = 0, ABRB_VEL_LINEAR = 1 };
enum {
  ABRB_PATH_ZERO_DISTANCE = -1, /* start == target (or a non-finite distance) */
  ABRB_PATH_OPPOSITE = -2,      /* target - start points exactly away from (1, 1, 1): align_vectors divides by 0 */
  ABRB_PATH_NO_VELOCITY = -3,   /* the max_v search reached 0 without fitting the ramps into the curve */
  ABRB_PATH_SHORT_RAMP = -4,    /* a velocity ramp of fewer than two samples */
  ABRB_PATH_TOO_LONG = -5       /* a ramp or the constant segment has 2^28 or more steps (or a non-finite count) */
};
typedef struct abrb_path_params {
  int32_t vel_kind;     /* ABRB_VEL_GAUSSIAN or ABRB_VEL_LINEAR, else ABRB_EUNSUP */
  int32_t n_points;     /* rows of table: 2 .. ABRB_PATH_MAX_POINTS (above: ABRB_EUNSUP) */
  double dt;            /* > 0 */
  double acceleration;  /* > 0 */
  double n_sigma;       /* > 0, Gaussian only */
  int32_t axes[4];      /* (firstaxis 0..2, parity, repetition, frame 0/1) of the Euler axes string, else ABRB_EUNSUP */
} abrb_path_params;
typedef struct abrb_path_rec {
  double max_v;         /* the velocity the search settled on */
  int32_t n_start, n_const, n_end;  /* samples of the starting ramp, the constant segment and the ending ramp */
  int32_t flags;        /* bit 0: start_velocity == max_velocity (ramp [v dt]); bit 1: the same at the end */
} abrb_path_rec;

/* ABRB_EINVAL: NULL params or array, B < 0, dt / acceleration / n_sigma not > 0, n_points < 2, misaligned pointer. */
int abrb_path_plan(const abrb_path_params *p, const double *table, const double *start, const double *target,
                   const double *max_velocity, const double *start_velocity, const double *target_velocity,
                   int64_t *lengths, abrb_path_rec *plan, int64_t B, void *stream);
/* As abrb_path_plan, and ABRB_EINVAL for s_max < 0 or above 2^30, or only one of the orientations given. */
int abrb_path_fill_f64(const abrb_path_params *p, const double *table, const double *start, const double *target,
                       const double *start_velocity, const double *target_velocity, const double *start_orientation,
                       const double *target_orientation, const abrb_path_rec *plan, const int64_t *lengths,
                       int64_t s_max, double *path, int64_t B, void *stream);
int abrb_path_fill_f32(const abrb_path_params *p, const double *table, const double *start, const double *target,
                       const double *start_velocity, const double *target_velocity, const double *start_orientation,
                       const double *target_orientation, const abrb_path_rec *plan, const int64_t *lengths,
                       int64_t s_max, float *path, int64_t B, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* ABRB_H_ */
