// kernels.cu — sm_90a kernels of the batched arm engine, compiled once per joint count (-DABRB_N=<n>).
//
// Mapping: ONE JOINT STATE PER THREAD.  The per-state arithmetic (abrb_math.cuh / abrb_rbd.cuh /
// abrb_osc.cuh) is a straight-line, fully unrolled sequence on registers; chain constants come from the
// kernel-parameter constant bank (uniform across the warp).  Loads of the (B, n) state arrays are
// contiguous per warp; every output array is staged per warp in shared memory and written back with
// fully coalesced 16-byte stores, so HBM sees whole 128-byte lines only.
#include <cuda_runtime.h>
#include <type_traits>
#include <utility>

#include <atomic>

#include "abrb_coop.cuh"
#include "abrb_grad.cuh"
#include "abrb_launch.hpp"
#include "abrb_osc.cuh"
#include "abrb_path.cuh"
#include "abrb_rbd.cuh"
#include "abrb_regress.cuh"

#ifndef ABRB_N
#error "compile with -DABRB_N=<joint count>"
#endif

namespace abrb {

namespace {

// CTA size of every kernel.  What ends the OSC kernel is the CTA whose queue of deferred states happens to hold more
// records than it has groups (a second Jacobi pass); 128 threads give a CTA 20 six-lane groups, 64 would give it half
// as many per queue.  256 threads do not fit the non-orthonormal fp64 scratch, and for the orthonormal fp64 kernels (54 scratch
// slots per lane) the evaluation gets slower by about as much as the flush gets cheaper.
constexpr int kBlock = 128;
// CTAs per SM the register allocator must allow: the fp64 kernels get the full 255 registers (2 CTAs/SM; capping them
// spills), the fp32 kernels 4 CTAs/SM (128 registers).
template <typename T>
struct MinBlocks {
  static constexpr int value = sizeof(T) == 8 ? 2 : 4;
};
constexpr int kWarps = kBlock / 32;

template <int N>
struct MaxRecord {
  static constexpr int big = N * N > 6 * N ? N * N : 6 * N;
  static constexpr int value = big > 16 ? big : 16;
};

// Per-warp shared-memory region: holds the warp's kinematic scratch (slot-major, stride 32: lane i owns column i,
// conflict-free) while a state is being evaluated and is then re-used as the staging tile for the coalesced
// stores.  The fp64 kernels keep the scratch in shared memory, which is what lets the plain OSC kernels (osc_plain) fit
// 255 registers without local-memory spills; the fp32 kernels keep it in registers and need only the staging tile.
template <typename T, int N, bool ORTHO>
struct KinSel;
template <int N, bool ORTHO>
struct KinSel<float, N, ORTHO> {
  typedef Kin<float, N, ORTHO, RegStore> type;
  static constexpr int kSlots = 0;
  static __device__ __forceinline__ void bind(type &, float *, int) {}
};
template <int N, bool ORTHO>
struct KinSel<double, N, ORTHO> {
  typedef Kin<double, N, ORTHO, StridedStore> type;
  static constexpr int kSlots = KinSlots<N, ORTHO>::kCount;
  static __device__ __forceinline__ void bind(type &k, double *warp_region, int lane) {
    k.s.base = warp_region + lane;
    k.s.stride = 32;
  }
};
template <int A, int B>
struct MaxI {
  static constexpr int value = A > B ? A : B;
};

// Write one LEN-element record per lane to `out[(warp_b0 + lane) * LEN + e]` through the warp's staging tile.
// The tile is element-major with a row pitch of 33 (`tile[e * 33 + lane]`): the per-lane writes are conflict-free
// (consecutive lanes -> consecutive words) and so are the reads of the linear copy-out (consecutive output
// elements -> pitch 33 -> distinct banks); the copy-out itself is perfectly coalesced (each warp instruction
// writes 32 consecutive elements = whole 128-byte lines).
constexpr int kPitch = 33;
// Records longer than kChunk elements go through the tile in slices of kChunk (the tile then needs only
// kPitch * kChunk elements per warp, which is what lets three CTAs of the fp64 kernels share an SM); each slice is a
// run of kChunk contiguous elements per record in global memory (>= 144 bytes for fp64).  STRIDE > LEN stores a part of
// a longer record (`out` then points at the part's first element in record 0).
constexpr int kChunk = 64;  // no slicing needed with 2 CTAs/SM (93 KB each); 18 would allow 3 CTAs/SM but measured slower
template <typename T, int LEN, int STRIDE = LEN>
__device__ __forceinline__ void store_records(T *__restrict__ out, int64_t warp_b0, int nvalid, const T *rec,
                                              T *tile, int lane) {
  T *dst = out + warp_b0 * STRIDE;
#pragma unroll
  for (int c0 = 0; c0 < LEN; c0 += kChunk) {
    constexpr int kFull = kChunk;
    const int ch = LEN - c0 < kFull ? LEN - c0 : kFull;  // compile-time after unrolling
    __syncwarp();
#pragma unroll
    for (int e = 0; e < kChunk; ++e)
      if (e < ch) tile[e * kPitch + lane] = rec[c0 + e];
    __syncwarp();
    const int total = nvalid * ch;
#pragma unroll
    for (int it = 0; it < kChunk; ++it) {
      if (it < ch) {
        const int i = it * 32 + lane;
        const int r = i / ch, e = i - r * ch;
        if (i < total) dst[r * STRIDE + c0 + e] = tile[e * kPitch + r];
      }
    }
  }
}

// Output functor handed to rbd_state: stores each finished record immediately (keeps the live register set small)
template <typename T>
struct RbdSink {
  T *ptr[kOutCount];
  T *tile;
  int64_t warp_b0;
  int nvalid, lane;
  template <int LEN>
  __device__ __forceinline__ void put(int which, const T *rec) {
    if (ptr[which] != nullptr) store_records<T, LEN>(ptr[which], warp_b0, nvalid, rec, tile, lane);
  }
};

template <typename T>
struct RbdArgs {
  const T *q, *dq;
  T *Tx, *Tm, *R, *Tinv, *quat, *J, *dJ, *M, *g, *C;
  int64_t B;
  int frame;
  unsigned want;
  T xoff[3];
};

// shared memory per warp: [ kinematic scratch (fp64 only): kSlots x 32 ][ staging tile: kPitch x max record ]
//                        [ exchange area of the cooperative pseudo-inverse (OSC kernels only): XCH x 32 ]
template <typename T, int N, bool ORTHO, int MAXREC, int XCH = 0>
struct WarpSmem {
  static constexpr int kKin = 32 * KinSel<T, N, ORTHO>::kSlots;
  static constexpr int kTile = kPitch * (MAXREC < kChunk ? MAXREC : kChunk);
  static constexpr int kXch = 32 * XCH;
  static constexpr int kElems = kKin + kTile + kXch;
};
template <typename T, int N, bool ORTHO, int KD>
struct OscSmem : WarpSmem<T, N, ORTHO, (N > 6 ? N : 6),
                          CoopLayout<N, KD, !KinSel<T, N, ORTHO>::type::kSharedScratch>::kSlots> {};

// Programmatic dependent launch (see launch_pdl): let the stream's next kernel be scheduled as CTAs of this one retire,
// and wait until the previous kernel of the stream has completed and its memory is visible.  Both are no-ops for a
// launch without the attribute.
__device__ __forceinline__ void pdl_entry() {
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename T, int N, bool ORTHO, bool DYN, bool CMAT, bool XTRA>
__global__ void __launch_bounds__(kBlock, MinBlocks<T>::value)
rbd_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ RbdArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef WarpSmem<T, N, ORTHO, MaxRecord<N>::value> WS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  typename KS::type K;
  KS::bind(K, region, lane);
  RbdSink<T> sink;
  sink.ptr[kOutTx] = a.Tx;
  sink.ptr[kOutT] = a.Tm;
  sink.ptr[kOutR] = a.R;
  sink.ptr[kOutTinv] = a.Tinv;
  sink.ptr[kOutQuat] = a.quat;
  sink.ptr[kOutJ] = a.J;
  sink.ptr[kOutdJ] = a.dJ;
  sink.ptr[kOutM] = a.M;
  sink.ptr[kOutg] = a.g;
  sink.ptr[kOutC] = a.C;
  sink.tile = region + WS::kKin;
  sink.lane = lane;
  pdl_entry();
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    // no early exit: every thread of the CTA takes part in the phase barriers; idle lanes / warps redo a valid state
    const int64_t warp_b0 = base + warp * 32;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (rem > 0 ? (int)rem : 0) : 32;
    const int64_t bb = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    const int64_t b = bb < a.B ? (bb >= 0 ? bb : 0) : a.B - 1;
    T q[N], dq[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq != nullptr ? a.dq[b * N + k] : T(0);
    }
    sink.warp_b0 = warp_b0;
    sink.nvalid = nvalid;
    rbd_state<T, N, DYN, CMAT, XTRA>(P, q, dq, a.frame, a.xoff, a.want, K, sink);
  }
}

template <typename T>
struct OscArgs {
  const T *q, *dq, *target, *tv;
  T *u, *train;
  T *ierr;  // (B, 6) integrated task-space error, updated in place (ki != 0), or nullptr
  int64_t B;
  int target_stride, tv_stride;
  GatherArgs g;  // n_peer > 0: also store u into every rank's gathered array (peer memory over NVLink)
  int *sched;    // {next tile, CTAs done} of this launch (zero on entry, re-armed by the last CTA), or nullptr: static tiles
};

// CTA-level shared memory of the OSC kernel behind the per-warp regions: the queue of deferred states (abrb_coop.cuh)
template <typename T, int N, int KD, int CAP>
struct OscQueue {
  static constexpr int kRecElems = CAP * CoopRecord<N, KD>::kLen;
  static constexpr size_t kRowOff = ((size_t)kRecElems * sizeof(T) + 15) / 16 * 16;   // long long rows[CAP]
  static constexpr size_t kCountOff = kRowOff + CAP * sizeof(long long);             // int count
  static constexpr size_t kBytes = kCountOff + 32;  // count (int), next tile (long long)
};

// One pass over the batch, persistent CTAs (grid = resident CTAs, tiles from a per-launch counter).  The states whose
// task-space inertia needs the truncating pseudo-inverse (3.8 % of uniformly random UR5 6-DOF states: 70 % of the warps
// hold one) leave a record in the CTA's queue and are finished by the whole CTA cooperatively (abrb_coop.cuh) once as
// many as the CTA has groups (20 or 16) have gathered or the CTA has run out of tiles; what does not fit the queue is
// finished by its warp in line.

// Resident CTAs per SM the OSC kernel is compiled for.  fp64: 2 (255 registers).  fp32 with orthonormal frames (UR5: the
// signed-permutation constants fold away): 4 (128 registers) measured best; fp32 with general frames (Jaco2) spills
// ~3 KB per thread at 128 registers, so it runs 2 CTAs at 255 registers.
template <typename T, bool ORTHO>
struct MinBlocksOsc {
  static constexpr int value = sizeof(T) == 8 || ORTHO ? MinBlocks<T>::value : 2;
};

// PLAIN: the instantiation for calls that qualify under osc_plain (abrb_host.hpp); see osc_eval.
template <typename T, int N, bool ORTHO, int KD, bool PLAIN>
__global__ void __launch_bounds__(kBlock, MinBlocksOsc<T, ORTHO>::value)
osc_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ OscK<T, N> O,
           const __grid_constant__ OscArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef OscSmem<T, N, ORTHO, KD> WS;
  constexpr int kOscFlushAt = kWarps * CoopGroup<N, KD>::kPerWarp;  // one full round of the CTA's groups
  constexpr int kCoopQueue = kCoopQueuePerWarp * kWarps;
  typedef OscQueue<T, N, KD, kCoopQueue> Q;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  T *stage = region + WS::kKin;
  unsigned char *qbase = smem_raw + ((size_t)kWarps * WS::kElems * sizeof(T) + 15) / 16 * 16;
  T *qrec = reinterpret_cast<T *>(qbase);
  long long *qrow = reinterpret_cast<long long *>(qbase + Q::kRowOff);
  int *qcount = reinterpret_cast<int *>(qbase + Q::kCountOff);
  if (threadIdx.x == 0) *qcount = 0;
  __syncthreads();
  typename KS::type K;
  KS::bind(K, region, lane);
  K.s.psync = sizeof(T) == 8;  // CTA phase barriers (abrb_math.cuh, RegStore::sync) pay in fp64 only, here and in rollout
  WarpCoop<T, N, KD, typename KS::type> coop{region + WS::kKin + WS::kTile, region, lane, true, qrec, qrow, qcount, 0,
                                             kCoopQueue};
  FlushOut<T> fo;
  fo.u = a.u;
  fo.train = a.train;
  fo.n_peer = a.g.n_peer;
  fo.self = a.g.self;
  fo.row0 = a.g.row0;
#pragma unroll
  for (int p = 0; p < kMaxPeers; ++p) fo.peer[p] = static_cast<T *>(a.g.peer_u[p]);
  const double rcond = double(O.thr) * 0.1;
  // Programmatic dependent launch: everything above touched only kernel parameters and shared memory.  A launch that
  // follows another kernel in its stream is allowed onto the SMs while that kernel's last CTAs are still running (its
  // launch latency, parameter upload and CTA ramp-up overlap their tail) and waits HERE, before its first global access,
  // until that kernel has completed and its memory is visible.  Without the launch attribute both are no-ops.
  pdl_entry();
  // Tiles: the first one is the CTA's own index; the following ones come from the launch's tile counter, so that a CTA
  // whose tiles happen to be expensive (obstacle-active states, many pseudo-inverse states) simply takes fewer of them.
  const long long n_tiles = (a.B + kBlock - 1) / kBlock;
  long long *next_tile = reinterpret_cast<long long *>(qbase + Q::kCountOff + 8);
  for (long long tile = blockIdx.x; tile < n_tiles;) {
    const int64_t base = tile * kBlock;
    // (the next tile's index is asked for now and published at the end of this tile: the atomic's round trip hides
    // under the evaluation)
    long long upcoming = 0;
    if (threadIdx.x == 0) upcoming = a.sched != nullptr ? (long long)gridDim.x + atomicAdd(a.sched, 1) : tile + gridDim.x;
    // no early exit: every lane of a warp takes part in the cooperative steps; idle lanes / warps redo a valid state
    const int64_t warp_b0 = base + warp * 32;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (rem > 0 ? (int)rem : 0) : 32;
    const int64_t bb = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    const int64_t b = bb < a.B ? (bb >= 0 ? bb : 0) : a.B - 1;
    T q[N], dq[N], tg[6], tv[6], ie[6], u[N], tr[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      tg[c] = a.target[b * a.target_stride + c];
      tv[c] = !PLAIN && a.tv != nullptr ? a.tv[b * a.tv_stride + c] : T(0);
      ie[c] = !PLAIN && a.ierr != nullptr ? a.ierr[b * 6 + c] : T(0);
    }
    coop.valid = lane < nvalid;
    coop.row = b;
    osc_eval<T, N, KD, false, PLAIN>(P, O, q, dq, tg, a.tv != nullptr ? tv : nullptr, a.ierr != nullptr ? ie : nullptr, u, tr,
                              (T *)nullptr, K, coop);
    if (a.u) store_records<T, N>(a.u, warp_b0, nvalid, u, stage, lane);
    if (a.train) store_records<T, N>(a.train, warp_b0, nvalid, tr, stage, lane);
    if (!PLAIN && a.ierr) store_records<T, 6>(a.ierr, warp_b0, nvalid, ie, stage, lane);
    // fused all-gather: this tile's rows go to every rank's gathered array while the other warps still compute
    for (int p = 0; p < a.g.n_peer; ++p)
      store_records<T, N>(static_cast<T *>(a.g.peer_u[p]), a.g.row0 + warp_b0, nvalid, u, stage, lane);
    // deferred states: emptied once a full round of the CTA's groups has gathered, and after the last tile
    if (threadIdx.x == 0) *next_tile = upcoming;
    __syncthreads();  // this tile's rows and records, and the next tile's index, are visible to the whole CTA
    const int queued = *qcount < kCoopQueue ? *qcount : kCoopQueue;
    tile = *next_tile;
    const bool last = tile >= n_tiles;
    if (queued >= kOscFlushAt || (last && queued > 0)) {
      coop_flush_cta<T, N, KD>(qrec, qrow, queued, fo, rcond, !PLAIN && O.n_null > 0);
      __syncthreads();
      if (threadIdx.x == 0) *qcount = 0;
    }
    __syncthreads();
  }
  if (a.sched != nullptr && threadIdx.x == 0) {  // every CTA has taken its last tile index: the last one re-arms the counter
    const int done = atomicAdd(a.sched + 1, 1);
    if (done == (int)gridDim.x - 1) {
      a.sched[0] = 0;
      a.sched[1] = 0;
      __threadfence();
    }
  }
  if (a.g.n_peer > 0) {
    // completion: once every CTA's peer stores are visible system-wide, the last CTA publishes this launch's epoch
    // in every rank's flag array; abrb_gather_wait() on the consumer side spins on those flags
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned done = atomicAdd(a.g.cta_counter, 1u);
      if (done == gridDim.x - 1) {
        *a.g.cta_counter = 0u;
        __threadfence_system();
        for (int p = 0; p < a.g.n_peer; ++p)
          asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(a.g.peer_flag[p]), "l"(a.g.epoch) : "memory");
      }
    }
  }
}

template <typename T>
struct RolloutArgs {
  T *q, *dq;
  const T *target;
  T *q_traj, *dq_traj, *u_traj;
  T *ierr;  // (B, 6) integrated task-space error, in/out (ki != 0), or nullptr
  int64_t B;
  int target_stride, steps;
  T dt;
};

// Path-following rollout: `target` is the path, element (t, b, c) at target[(t B + b) 6 + c] when target_stride == 6
// (one path per trajectory) or at target[t 6 + c] when 0 (one path shared by every trajectory); `tv` likewise.
template <typename T>
struct RolloutPathArgs : RolloutArgs<T> {
  const T *tv;       // path velocity, or nullptr
  T *x_traj, *cost;  // (steps, B, 3) control-point track, (B,) tracking cost, or nullptr
  int tv_stride;
  T effort;          // weight of |u|^2 in the cost
};

// Closed loop: u = OSC(q, dq); ddq = M^-1 (u + g - C dq); dq += ddq dt; q += dq dt  (state stays in registers).
// Args = RolloutArgs: one fixed target per trajectory (abrb_osc_rollout_*).  Args = RolloutPathArgs: the target and
// target velocity of step t come from the path, and the control point of each step's state and the tracking cost are
// recorded too (abrb_osc_rollout_path_*).  (The two share this body as one kernel template: moving the loop into a
// device function of its own changes the generated code of the fixed-target instantiations.)
template <typename T, int N, bool ORTHO, int KD, bool PLAIN, class Args>
__global__ void __launch_bounds__(kBlock)
rollout_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ OscK<T, N> O,
               const __grid_constant__ Args a) {
  constexpr bool PATH = std::is_same<Args, RolloutPathArgs<T>>::value;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef OscSmem<T, N, ORTHO, KD> WS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  T *stage = region + WS::kKin;
  typename KS::type K;
  KS::bind(K, region, lane);
  K.s.psync = sizeof(T) == 8;
  WarpCoop<T, N, KD, typename KS::type> coop{region + WS::kKin + WS::kTile, region, lane, true};
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    // no early exit (cooperative step inside osc_eval): idle lanes / warps redo a valid state and store nothing
    const int64_t warp_b0 = base + warp * 32;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (rem > 0 ? (int)rem : 0) : 32;
    const int64_t bb = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    const int64_t b = bb < a.B ? (bb >= 0 ? bb : 0) : a.B - 1;
    T q[N], dq[N], tg[6], ie[6], u[N], tv[6], x[3];
    T cost = T(0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      if (!PATH) tg[c] = a.target[b * a.target_stride + c];
      ie[c] = !PLAIN && a.ierr != nullptr ? a.ierr[b * 6 + c] : T(0);
    }
    coop.valid = lane < nvalid;
    for (int t = 0; t < a.steps; ++t) {
      const T *tvp = nullptr;
      T effort = T(0);
      if constexpr (PATH) {
        // a shared path is one address for the whole warp (a broadcast load); a per-trajectory path is one row per lane
        const T *pt = path_row(a.target, a.target_stride, t, a.B, b);
#pragma unroll
        for (int c = 0; c < 6; ++c) tg[c] = pt[c];
        if (!PLAIN && a.tv != nullptr) {
          const T *vt = path_row(a.tv, a.tv_stride, t, a.B, b);
#pragma unroll
          for (int c = 0; c < 6; ++c) tv[c] = vt[c];
          tvp = tv;
        }
        effort = a.effort;
      }
      rollout_step<T, N, KD, PLAIN, PATH>(P, O, q, dq, tg, tvp, a.ierr != nullptr ? ie : nullptr, a.dt, effort, u, x,
                                          cost, K, coop);
      const int64_t row0 = (int64_t)t * a.B + warp_b0;
      if (a.u_traj) store_records<T, N>(a.u_traj, row0, nvalid, u, stage, lane);
      if (a.q_traj) store_records<T, N>(a.q_traj, row0, nvalid, q, stage, lane);
      if (a.dq_traj) store_records<T, N>(a.dq_traj, row0, nvalid, dq, stage, lane);
      if constexpr (PATH) {
        if (a.x_traj) store_records<T, 3>(a.x_traj, row0, nvalid, x, stage, lane);
      }
    }
    store_records<T, N>(a.q, warp_b0, nvalid, q, stage, lane);
    store_records<T, N>(a.dq, warp_b0, nvalid, dq, stage, lane);
    if (!PLAIN && a.ierr) store_records<T, 6>(a.ierr, warp_b0, nvalid, ie, stage, lane);
    if constexpr (PATH) {
      if (a.cost != nullptr && lane < nvalid) a.cost[b] = cost;
    }
  }
}

template <typename T>
struct NullArgs {
  const T *q, *dq;
  T *u;
  int64_t B;
};

template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
null_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ NullK<T, N> Z,
            const __grid_constant__ NullArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *stage = reinterpret_cast<T *>(smem_raw) + warp * kPitch * (N < kChunk ? N : kChunk);
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], u[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
    Kin<T, N, ORTHO> K;
    null_state<T, N>(P, Z, q, dq, u, K);
    store_records<T, N>(a.u, warp_b0, nvalid, u, stage, lane);
  }
}

template <typename T>
struct CtrlArgs {
  const T *q, *dq, *target, *tv;
  T *u;
  int64_t B;
  int target_stride, tv_stride, kind, flag_a, flag_b;
  T kp, kv;
};

// Joint.generate / Floating.generate: small relatives of the kernels above (M, g, one product or one 3x3 solve)
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
ctrl_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ CtrlArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *stage = reinterpret_cast<T *>(smem_raw) + warp * kPitch * N;
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], tg[N], tv[N], u[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq != nullptr ? a.dq[b * N + k] : T(0);
      tg[k] = a.target != nullptr ? a.target[b * a.target_stride + k] : T(0);
      tv[k] = a.tv != nullptr ? a.tv[b * a.tv_stride + k] : T(0);
    }
    Kin<T, N, ORTHO> K;
    if (a.kind == 0)
      joint_state<T, N>(P, a.kp, a.kv, a.flag_a != 0, q, dq, tg, a.tv != nullptr ? tv : nullptr, u, K);
    else
      floating_state<T, N>(P, a.flag_a != 0, a.flag_b != 0, q, dq, u, K);
    store_records<T, N>(a.u, warp_b0, nvalid, u, stage, lane);
  }
}

template <typename T>
struct SlidingArgs {
  const T *q, *dq, *target, *tv, *ta;
  T *u, *s;
  int64_t B;
  int target_stride, tv_stride, ta_stride, cartesian, frame;
  T kd, lamb;
  T xoff[3];
};

// Sliding.generate: J, dJ, M, C, g of one state and two applications of pinv(J) (abrb_osc.cuh, sliding_state)
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
sliding_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ SlidingArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *stage = reinterpret_cast<T *>(smem_raw) + warp * kPitch * N;
  const int w = a.cartesian ? 3 : N;
  constexpr int L = CtrlRow<N>::kMax;  // a cartesian row is 3 wide whatever N is
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], tg[L], tv[L], ta[L], u[N], sv[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
#pragma unroll
    for (int k = 0; k < L; ++k) {
      const bool on = k < w;
      tg[k] = on ? a.target[b * a.target_stride + k] : T(0);
      tv[k] = (on && a.tv != nullptr) ? a.tv[b * a.tv_stride + k] : T(0);
      ta[k] = (on && a.ta != nullptr) ? a.ta[b * a.ta_stride + k] : T(0);
    }
    Kin<T, N, ORTHO> K;
    sliding_state<T, N>(P, a.kd, a.lamb, a.cartesian != 0, a.frame, a.xoff, q, dq, tg, tv, ta, u, sv, K);
    store_records<T, N>(a.u, warp_b0, nvalid, u, stage, lane);
    if (a.s != nullptr) store_records<T, N>(a.s, warp_b0, nvalid, sv, stage, lane);
  }
}

template <typename T>
struct IkArgs {
  const T *position, *target;
  T *pos_path, *vel_path;  // (steps, B, n)
  int64_t B;
  int target_stride, steps, method;
  T max_dx, max_dr, max_dq;  // already multiplied by dt
};

// InverseKinematics.generate_path: one trajectory per thread, the joint state stays in registers over the steps
// (sequential by construction, like the rollout kernel)
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
ik_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ IkArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *stage = reinterpret_cast<T *>(smem_raw) + warp * kPitch * N;
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], tg[3], Qd[4];
#pragma unroll
    for (int k = 0; k < N; ++k) q[k] = a.position[b * N + k];
#pragma unroll
    for (int c = 0; c < 3; ++c) tg[c] = a.target[b * a.target_stride + c];
    quat_from_euler_sxyz(a.target[b * a.target_stride + 3], a.target[b * a.target_stride + 4],
                         a.target[b * a.target_stride + 5], Qd);
    const T nq = T(1) / sqrt_t(Qd[0] * Qd[0] + Qd[1] * Qd[1] + Qd[2] * Qd[2] + Qd[3] * Qd[3]);
#pragma unroll
    for (int i = 0; i < 4; ++i) Qd[i] *= nq;
    for (int t = 0; t < a.steps; ++t) {
      Kin<T, N, ORTHO> K;
      ik_step<T, N>(P, a.max_dx, a.max_dr, a.max_dq, a.method, q, tg, Qd, dq, K);
      const int64_t row0 = (int64_t)t * a.B + warp_b0;
      store_records<T, N>(a.pos_path, row0, nvalid, q, stage, lane);
      store_records<T, N>(a.vel_path, row0, nvalid, dq, stage, lane);
#pragma unroll
      for (int k = 0; k < N; ++k) q[k] += dq[k];
    }
  }
}

template <typename T>
struct PlantArgs {
  T *q, *dq;
  const T *u;     // torques, row t of trajectory b at torque_row(u, u_stride, t, B, b)
  const T *path;  // (steps, B, 6) (path_stride 6), (steps, 6) (0), or nullptr
  T *q_traj, *dq_traj, *u_traj, *x_traj, *cost;
  int64_t B;
  int u_stride, path_stride, steps, frame, comp_g;
  T dt, effort;
  T xoff[3];
};

// Open-loop plant rollout (abrb_plant_rollout_*): one trajectory per thread, q and dq in registers across the steps,
// the torque of step t read from the caller's sequence (plant_step, abrb_rbd.cuh).  M is factorised by Cholesky, so
// there is no cooperative part; the kinematic scratch is the one the rollout kernel uses.
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
plant_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ PlantArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef WarpSmem<T, N, ORTHO, (N > 3 ? N : 3)> WS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  T *stage = region + WS::kKin;
  typename KS::type K;
  KS::bind(K, region, lane);
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], ur[N], tau[N], x[3];
    T cost = T(0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
    for (int t = 0; t < a.steps; ++t) {
      // a shared sequence (or path) is one address for the whole warp (a broadcast load), a per-trajectory one a row
      // per lane
      const T *ut = torque_row<T, N>(a.u, a.u_stride, t, a.B, b);
#pragma unroll
      for (int k = 0; k < N; ++k) ur[k] = ut[k];
      const T *pt = a.path != nullptr ? path_row(a.path, a.path_stride, t, a.B, b) : nullptr;
      plant_step<T, N>(P, a.frame, a.xoff, q, dq, ur, a.comp_g != 0, pt, a.dt, a.effort, tau, x, cost, K);
      const int64_t row0 = (int64_t)t * a.B + warp_b0;
      if (a.u_traj) store_records<T, N>(a.u_traj, row0, nvalid, tau, stage, lane);
      if (a.q_traj) store_records<T, N>(a.q_traj, row0, nvalid, q, stage, lane);
      if (a.dq_traj) store_records<T, N>(a.dq_traj, row0, nvalid, dq, stage, lane);
      if (a.x_traj) store_records<T, 3>(a.x_traj, row0, nvalid, x, stage, lane);
    }
    store_records<T, N>(a.q, warp_b0, nvalid, q, stage, lane);
    store_records<T, N>(a.dq, warp_b0, nvalid, dq, stage, lane);
    if (a.cost != nullptr && lane < nvalid) a.cost[b] = cost;
  }
}

template <typename T>
struct CtrlRolloutArgs {
  T *q, *dq;
  const T *path, *pv, *pa;  // rows of width 3 (cartesian Sliding) or N at torque_row(.., stride, t, B, b); pv, pa may be
                            // nullptr (pa: Sliding only)
  T *q_traj, *dq_traj, *u_traj, *x_traj, *cost;
  int64_t B;
  int path_stride, pv_stride, pa_stride, steps, frame;
  CtrlK<T> G;
  T dt, effort;
  T xoff[3];
};

// Closed-loop Joint / Sliding rollout (abrb_joint_rollout_path_*, abrb_sliding_rollout_path_*): one trajectory per
// thread, q and dq in registers across the steps, the controller and the plant of each step in ctrl_rollout_step
// (abrb_osc.cuh).  Shaped like plant_kernel, with the same kinematic scratch.
template <typename T, int N, bool ORTHO, int KIND>
__global__ void __launch_bounds__(kBlock)
ctrl_rollout_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ CtrlRolloutArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef WarpSmem<T, N, ORTHO, (N > 3 ? N : 3)> WS;
  constexpr int L = CtrlRow<N>::kMax;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  T *stage = region + WS::kKin;
  typename KS::type K;
  KS::bind(K, region, lane);
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], tg[L], tv[L], ta[L], u[N], x[3];
    T cost = T(0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
    }
    for (int t = 0; t < a.steps; ++t) {
      // a shared path is one address for the whole warp (a broadcast load), a per-trajectory one a row per lane
      ctrl_path_rows<T, N, KIND>(a.path, a.path_stride, a.pv, a.pv_stride, a.pa, a.pa_stride, a.G.cartesian != 0, t,
                                 a.B, b, tg, tv, ta);
      ctrl_rollout_step<T, N, KIND>(P, a.G, a.frame, a.xoff, q, dq, tg, a.pv != nullptr ? tv : nullptr,
                                    a.pa != nullptr ? ta : nullptr, a.dt, a.effort, u, x, cost, K);
      const int64_t row0 = (int64_t)t * a.B + warp_b0;
      if (a.u_traj) store_records<T, N>(a.u_traj, row0, nvalid, u, stage, lane);
      if (a.q_traj) store_records<T, N>(a.q_traj, row0, nvalid, q, stage, lane);
      if (a.dq_traj) store_records<T, N>(a.dq_traj, row0, nvalid, dq, stage, lane);
      if (a.x_traj) store_records<T, 3>(a.x_traj, row0, nvalid, x, stage, lane);
    }
    store_records<T, N>(a.q, warp_b0, nvalid, q, stage, lane);
    store_records<T, N>(a.dq, warp_b0, nvalid, dq, stage, lane);
    if (a.cost != nullptr && lane < nvalid) a.cost[b] = cost;
  }
}

template <typename T>
struct DynArgs {
  const T *q, *dq, *in;  // in: u (kind 0) or ddq (kind 1)
  T *out;                // ddq (kind 0) or u (kind 1)
  int64_t B;
  int kind;
};

// abrb_forward_dynamics_* (kind 0) and abrb_inverse_dynamics_* (kind 1): one state per thread, grid-stride
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
dyn_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ DynArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef WarpSmem<T, N, ORTHO, N> WS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  T *stage = region + WS::kKin;
  typename KS::type K;
  KS::bind(K, region, lane);
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], in[N], out[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
      in[k] = a.in[b * N + k];
    }
    if (a.kind == 0)
      forward_dynamics_state<T, N>(P, q, dq, in, out, K);
    else
      inverse_dynamics_state<T, N>(P, q, dq, in, out, K);
    store_records<T, N>(a.out, warp_b0, nvalid, out, stage, lane);
  }
}

template <typename T>
struct RegressorArgs {
  const T *q, *dq, *ddq;
  T *Yt;  // (B, 6N, N)
  int64_t B;
  T gravity[6];
};

// Output functor handed to inverse_dynamics_regressor: stores each finished half of a state's record at once
template <typename T, int N>
struct RegressorSink {
  T *Yt, *tile;
  int64_t warp_b0;
  int nvalid, lane;
  template <int LEN>
  __device__ __forceinline__ void put(int off, const T *rec) {
    store_records<T, LEN, RegressorLayout<N>::kRecord>(Yt + off, warp_b0, nvalid, rec, tile, lane);
  }
};

// abrb_inverse_dynamics_regressor_*: one state per thread, grid-stride.  A state reads 3N values and writes 6N^2.
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(kBlock)
regressor_kernel(const __grid_constant__ ChainK<T, N> P, const __grid_constant__ RegressorArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef KinSel<T, N, ORTHO> KS;
  typedef WarpSmem<T, N, ORTHO, RegressorLayout<N>::kHalf> WS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T *region = reinterpret_cast<T *>(smem_raw) + warp * WS::kElems;
  typename KS::type K;
  KS::bind(K, region, lane);
  RegressorSink<T, N> sink;
  sink.Yt = a.Yt;
  sink.tile = region + WS::kKin;
  sink.lane = lane;
  for (int64_t base = (int64_t)blockIdx.x * kBlock; base < a.B; base += (int64_t)gridDim.x * kBlock) {
    const int64_t warp_b0 = base + warp * 32;
    if (warp_b0 >= a.B) break;
    const int64_t rem = a.B - warp_b0;
    const int nvalid = rem < 32 ? (int)rem : 32;
    const int64_t b = warp_b0 + (lane < nvalid ? lane : nvalid - 1);
    T q[N], dq[N], ddq[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
      ddq[k] = a.ddq[b * N + k];
    }
    sink.warp_b0 = warp_b0;
    sink.nvalid = nvalid;
    inverse_dynamics_regressor<T, N>(P, a.gravity, q, dq, ddq, sink, K);
  }
}

// ------------------------------------------------------------------------------------------------ derivatives
// The derivative kernels run one warp per state (dyn_jac_kernel) or per trajectory (plant_vjp_kernel); lane j < 3N
// pushes direction j of the inputs through one dual evaluation (abrb_grad.cuh), and the other lanes idle.  The dual
// kinematic scratch (16 B a slot in fp64) lives in shared memory, one column per working lane (stride 3N); CTAs are
// 128 threads for orthonormal chains and 64 for general frames, whose scratch is 21 N slots instead of 9 N.
template <bool ORTHO>
struct DualBlock {
  static constexpr int value = ORTHO ? 128 : 64;
};
template <typename T, int N, bool ORTHO>
struct DualSmem {
  static constexpr size_t kWarpBytes = (size_t)3 * N * KinSlots<N, ORTHO>::kCount * sizeof(Dual<T>);
  static constexpr size_t kBytes = kWarpBytes * (DualBlock<ORTHO>::value / 32);
};

template <typename T, int N, bool ORTHO>
__device__ __forceinline__ void bind_dual_kin(Kin<Dual<T>, N, ORTHO, StridedStore> &K, unsigned char *smem, int warp,
                                              int lane) {
  K.s.base = reinterpret_cast<Dual<T> *>(smem + warp * DualSmem<T, N, ORTHO>::kWarpBytes) + lane;
  K.s.stride = 3 * N;
}

template <typename T>
struct DynJacArgs {
  const T *q, *dq, *in;
  T *d_q, *d_dq, *d_in;
  int64_t B;
  int kind;
};

// abrb_{forward,inverse}_dynamics_derivatives_*: lane j writes column j of the state's three n x n blocks, so each
// store instruction of a warp covers whole contiguous rows of a block
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(DualBlock<ORTHO>::value)
dyn_jac_kernel(const __grid_constant__ ChainK<Dual<T>, N> P, const __grid_constant__ DynJacArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Kin<Dual<T>, N, ORTHO, StridedStore> K;
  bind_dual_kin<T, N, ORTHO>(K, smem_raw, warp, lane);
  const int ncol = a.d_in != nullptr ? 3 * N : 2 * N;
  for (int64_t b = (int64_t)blockIdx.x * kW + warp; b < a.B; b += (int64_t)gridDim.x * kW) {
    if (lane >= ncol) continue;
    T q[N], dq[N], in[N], col[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      q[k] = a.q[b * N + k];
      dq[k] = a.dq[b * N + k];
      in[k] = a.in[b * N + k];
    }
    dyn_jac_column<T, N>(P, a.kind, lane, q, dq, in, col, K);
    T *dst = lane < N ? a.d_q : (lane < 2 * N ? a.d_dq : a.d_in);
    const int c = lane < N ? lane : (lane < 2 * N ? lane - N : lane - 2 * N);
#pragma unroll
    for (int i = 0; i < N; ++i) dst[(b * N + i) * N + c] = col[i];
  }
}

template <typename T>
struct PlantVjpArgs {
  const T *q0, *dq0, *u, *path, *q_traj, *dq_traj;
  const T *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  T *gu, *gq0, *gdq0;
  int64_t B;
  int u_stride, path_stride, steps, frame, comp_g;
  T dt, effort;
  T xoff[3];
};

// abrb_plant_rollout_vjp_*: the adjoint recursion of the rollout, t = S-1 .. 0, one warp per trajectory.  Every lane
// holds mu (the cotangent of x_{t+1}); lane j < 3N computes its entry of lambda_t (j < 2N) or of the torque cotangent
// (j >= 2N, stored), and lambda_t is broadcast with shuffles as the next step's mu.  No per-step Jacobian is stored.
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(DualBlock<ORTHO>::value)
plant_vjp_kernel(const __grid_constant__ ChainK<Dual<T>, N> P, const __grid_constant__ PlantVjpArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Kin<Dual<T>, N, ORTHO, StridedStore> K;
  bind_dual_kin<T, N, ORTHO>(K, smem_raw, warp, lane);
  const Dual<T> xo[3] = {Dual<T>(a.xoff[0]), Dual<T>(a.xoff[1]), Dual<T>(a.xoff[2])};
  for (int64_t b = (int64_t)blockIdx.x * kW + warp; b < a.B; b += (int64_t)gridDim.x * kW) {
    T mu[2 * N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      mu[k] = a.g_q != nullptr ? a.g_q[b * N + k] : T(0);
      mu[N + k] = a.g_dq != nullptr ? a.g_dq[b * N + k] : T(0);
    }
    const T gc = a.g_cost != nullptr ? a.g_cost[b] : T(0);
    for (int t = a.steps - 1; t >= 0; --t) {
      const int64_t row = (int64_t)t * a.B + b;
      if (a.g_q_traj != nullptr) {
#pragma unroll
        for (int k = 0; k < N; ++k) mu[k] += a.g_q_traj[row * N + k];
      }
      if (a.g_dq_traj != nullptr) {
#pragma unroll
        for (int k = 0; k < N; ++k) mu[N + k] += a.g_dq_traj[row * N + k];
      }
      T val = T(0);
      if (lane < 3 * N) {
        const T *qs = t > 0 ? a.q_traj + (row - a.B) * N : a.q0 + b * N;
        const T *dqs = t > 0 ? a.dq_traj + (row - a.B) * N : a.dq0 + b * N;
        T q[N], dq[N], ur[N], pr[3];
        const T *ut = torque_row<T, N>(a.u, a.u_stride, t, a.B, b);
#pragma unroll
        for (int k = 0; k < N; ++k) {
          q[k] = qs[k];
          dq[k] = dqs[k];
          ur[k] = ut[k];
        }
        if (a.path != nullptr) {
          const T *pt = path_row(a.path, a.path_stride, t, a.B, b);
#pragma unroll
          for (int c = 0; c < 3; ++c) pr[c] = pt[c];
        }
        val = plant_vjp_lane<T, N>(P, a.frame, xo, lane, q, dq, ur, a.comp_g != 0, a.path != nullptr ? pr : nullptr,
                                   a.dt, a.effort, mu, gc, a.g_x_traj != nullptr ? a.g_x_traj + row * 3 : nullptr,
                                   a.g_u_traj != nullptr ? a.g_u_traj + row * N : nullptr, K);
        if (lane >= 2 * N) a.gu[row * N + lane - 2 * N] = val;
      }
#pragma unroll
      for (int k = 0; k < 2 * N; ++k) mu[k] = __shfl_sync(0xffffffffu, val, k);
    }
    if (lane < N)
      a.gq0[b * N + lane] = mu[lane];
    else if (lane < 2 * N)
      a.gdq0[b * N + lane - N] = mu[lane];
  }
}

// The Joint closed loop's vector-Jacobian product has 4N + 2 working lanes (joint_vjp_lane): its dual kinematic
// scratch is one column per working lane, (4N + 2) x KinSlots per warp, in CTAs of DualBlock<ORTHO> threads (UR5,
// orthonormal: 22.5 KB a warp; a general 7-joint chain: 70.5 KB a warp).
template <typename T, int N, bool ORTHO>
struct JointDualSmem {
  static constexpr int kCols = 4 * N + 2;
  static constexpr size_t kWarpBytes = (size_t)kCols * KinSlots<N, ORTHO>::kCount * sizeof(Dual<T>);
  static constexpr size_t kBytes = kWarpBytes * (DualBlock<ORTHO>::value / 32);
};

template <typename T>
struct JointVjpArgs {
  const T *q0, *dq0, *path, *pv, *q_traj, *dq_traj;
  const T *g_cost, *g_q, *g_dq, *g_q_traj, *g_dq_traj, *g_u_traj, *g_x_traj;
  T *g_path, *g_pv, *g_gains, *gq0, *gdq0;  // g_path, g_pv, g_gains may be nullptr (not wanted)
  int64_t B;
  int path_stride, pv_stride, steps, frame, gravity;
  T kp, kv, dt, effort;
  T xoff[3];
};

// abrb_joint_rollout_path_vjp_*: the adjoint recursion of the Joint closed loop, t = S-1 .. 0, one warp per trajectory,
// shaped like plant_vjp_kernel.  Every lane holds mu; lanes j < 2N compute lambda_t, lanes 2N..4N-1 the path and path
// velocity cotangents of step t (stored per step), lanes 4N and 4N + 1 accumulate the gain cotangents over the steps
// (stored once).  Lanes whose output is not wanted idle.
template <typename T, int N, bool ORTHO>
__global__ void __launch_bounds__(DualBlock<ORTHO>::value)
joint_vjp_kernel(const __grid_constant__ ChainK<Dual<T>, N> P, const __grid_constant__ JointVjpArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef JointDualSmem<T, N, ORTHO> S;
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Kin<Dual<T>, N, ORTHO, StridedStore> K;
  K.s.base = reinterpret_cast<Dual<T> *>(smem_raw + warp * S::kWarpBytes) + lane;
  K.s.stride = S::kCols;
  const Dual<T> xo[3] = {Dual<T>(a.xoff[0]), Dual<T>(a.xoff[1]), Dual<T>(a.xoff[2])};
  const bool work = lane < 2 * N || (lane < 3 * N && a.g_path != nullptr) || (lane < 4 * N && lane >= 3 * N &&
                    a.g_pv != nullptr) || (lane >= 4 * N && lane < S::kCols && a.g_gains != nullptr);
  for (int64_t b = (int64_t)blockIdx.x * kW + warp; b < a.B; b += (int64_t)gridDim.x * kW) {
    T mu[2 * N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      mu[k] = a.g_q != nullptr ? a.g_q[b * N + k] : T(0);
      mu[N + k] = a.g_dq != nullptr ? a.g_dq[b * N + k] : T(0);
    }
    const T gc = a.g_cost != nullptr ? a.g_cost[b] : T(0);
    T gain = T(0);
    for (int t = a.steps - 1; t >= 0; --t) {
      const int64_t row = (int64_t)t * a.B + b;
      if (a.g_q_traj != nullptr) {
#pragma unroll
        for (int k = 0; k < N; ++k) mu[k] += a.g_q_traj[row * N + k];
      }
      if (a.g_dq_traj != nullptr) {
#pragma unroll
        for (int k = 0; k < N; ++k) mu[N + k] += a.g_dq_traj[row * N + k];
      }
      T val = T(0);
      if (work) {
        const T *qs = t > 0 ? a.q_traj + (row - a.B) * N : a.q0 + b * N;
        const T *dqs = t > 0 ? a.dq_traj + (row - a.B) * N : a.dq0 + b * N;
        const T *pt = torque_row<T, N>(a.path, a.path_stride, t, a.B, b);
        const T *vt = a.pv != nullptr ? torque_row<T, N>(a.pv, a.pv_stride, t, a.B, b) : nullptr;
        T q[N], dq[N], pr[N], vr[N];
#pragma unroll
        for (int k = 0; k < N; ++k) {
          q[k] = qs[k];
          dq[k] = dqs[k];
          pr[k] = pt[k];
          vr[k] = vt != nullptr ? vt[k] : T(0);
        }
        val = joint_vjp_lane<T, N>(P, a.kp, a.kv, a.gravity != 0, a.frame, xo, lane, q, dq, pr,
                                   vt != nullptr ? vr : nullptr, a.dt, a.effort, mu, gc,
                                   a.g_x_traj != nullptr ? a.g_x_traj + row * 3 : nullptr,
                                   a.g_u_traj != nullptr ? a.g_u_traj + row * N : nullptr, K);
        if (lane >= 2 * N && lane < 3 * N)
          a.g_path[row * N + lane - 2 * N] = val;
        else if (lane >= 3 * N && lane < 4 * N)
          a.g_pv[row * N + lane - 3 * N] = val;
        else if (lane >= 4 * N)
          gain += val;
      }
#pragma unroll
      for (int k = 0; k < 2 * N; ++k) mu[k] = __shfl_sync(0xffffffffu, val, k);
    }
    if (lane < N)
      a.gq0[b * N + lane] = mu[lane];
    else if (lane < 2 * N)
      a.gdq0[b * N + lane - N] = mu[lane];
    else if (lane >= 4 * N && lane < S::kCols && a.g_gains != nullptr)
      a.g_gains[b * 2 + lane - 4 * N] = gain;
  }
}

// ------------------------------------------------------------------------------------------------ launch
// kernel<<<grid, block, smem, stream>>>(args...) with programmatic stream serialization allowed: the launch may be
// brought onto the SMs while the stream's previous kernel drains; the kernels launched through it (osc_kernel,
// rbd_kernel) call pdl_entry() before their first global-memory access, which holds them until that kernel has
// completed and flushed.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t stream,
                              Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

inline int num_sms() {
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0)
      sm_count = 132;
  }
  return sm_count;
}

inline int grid_for(int64_t B, int blocks_per_sm) {
  const int64_t tiles = (B + kBlock - 1) / kBlock;
  const int64_t cap = (int64_t)num_sms() * blocks_per_sm;
  return (int)(tiles < cap ? tiles : cap);
}

template <typename K>
inline cudaError_t set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return cudaSuccess;
}

template <typename T, int N, bool ORTHO, bool DYN, bool CMAT, bool XTRA>
int rbd_go(const ChainHost &h, const RbdCall &c, unsigned want) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  RbdArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.Tx = static_cast<T *>(c.out.Tx);
  a.Tm = static_cast<T *>(c.out.T);
  a.R = static_cast<T *>(c.out.R);
  a.Tinv = static_cast<T *>(c.out.T_inv);
  a.quat = static_cast<T *>(c.out.quat);
  a.J = static_cast<T *>(c.out.J);
  a.dJ = static_cast<T *>(c.out.dJ);
  a.M = static_cast<T *>(c.out.M);
  a.g = static_cast<T *>(c.out.g);
  a.C = static_cast<T *>(c.out.C);
  a.B = c.B;
  a.frame = c.frame;
  a.want = want;
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  const size_t smem = (size_t)kWarps * WarpSmem<T, N, ORTHO, MaxRecord<N>::value>::kElems * sizeof(T);
  auto kern = rbd_kernel<T, N, ORTHO, DYN, CMAT, XTRA>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  e = launch_pdl(kern, grid_for(c.B, 8), kBlock, smem, c.stream, P, a);
  count_launch();
  return e != cudaSuccess ? (int)e : (int)cudaGetLastError();
}

template <typename T, int N>
int rbd_dispatch(const ChainHost &h, const RbdCall &c) {
  unsigned want = 0;
  if (c.out.Tx) want |= kWantTx;
  if (c.out.T) want |= kWantT;
  if (c.out.R) want |= kWantR;
  if (c.out.T_inv) want |= kWantTinv;
  if (c.out.quat) want |= kWantQuat;
  if (c.out.J) want |= kWantJ;
  if (c.out.dJ) want |= kWantdJ | kWantJ;
  if (c.out.M) want |= kWantM;
  if (c.out.g) want |= kWantg;
  if (c.out.C) want |= kWantC;
  const bool cm = c.out.C != nullptr, dyn = c.out.M != nullptr || c.out.g != nullptr;
  const bool xtra = (want & ~(kWantJ | kWantM | kWantg | kWantC)) != 0;
  // instantiations: {frame-only (with extras)} + {dynamics / dynamics+C} x {with, without extras}
#define ABRB_RBD_GO(O_)                                                                   \
  do {                                                                                     \
    if (cm) return xtra ? rbd_go<T, N, O_, true, true, true>(h, c, want) : rbd_go<T, N, O_, true, true, false>(h, c, want);   \
    if (dyn) return xtra ? rbd_go<T, N, O_, true, false, true>(h, c, want) : rbd_go<T, N, O_, true, false, false>(h, c, want); \
    return rbd_go<T, N, O_, false, false, true>(h, c, want);                               \
  } while (0)
  if (h.ortho) ABRB_RBD_GO(true);
  ABRB_RBD_GO(false);
#undef ABRB_RBD_GO
}

template <typename T, int N, bool ORTHO, int KD, bool PLAIN>
int osc_launch(const ChainHost &h, const abrb_osc_params &p, const OscCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, c.frame, c.xoff, O);
  OscArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.target = static_cast<const T *>(c.target);
  a.tv = static_cast<const T *>(c.tv);
  a.u = static_cast<T *>(c.u);
  a.train = static_cast<T *>(c.train);
  a.ierr = static_cast<T *>(c.ierr);
  a.B = c.B;
  a.target_stride = c.target_stride;
  a.tv_stride = c.tv_stride;
  if (c.gather != nullptr) a.g = *c.gather;
  a.sched = c.sched;
  const size_t smem = ((size_t)kWarps * OscSmem<T, N, ORTHO, KD>::kElems * sizeof(T) + 15) / 16 * 16 +
                      OscQueue<T, N, KD, kCoopQueuePerWarp * kWarps>::kBytes;
  auto kern = osc_kernel<T, N, ORTHO, KD, PLAIN>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  // persistent CTAs: as many as are resident at once, so that each sees several tiles and its deferred states gather
  static thread_local int resident = 0;
  static thread_local int resident_dev = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (resident_dev != dev) {
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kBlock, smem);
    if (e != cudaSuccess) return (int)e;
    resident = per_sm > 0 ? per_sm : 1;
    resident_dev = dev;
  }
  const int64_t tiles = (c.B + kBlock - 1) / kBlock, cap = (int64_t)num_sms() * resident;
  e = launch_pdl(kern, (unsigned)(tiles < cap ? tiles : cap), kBlock, smem, c.stream, P, O, a);
  count_launch();
  return e != cudaSuccess ? (int)e : (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO, int KD>
int osc_go(const ChainHost &h, const abrb_osc_params &p, const OscCall &c) {
  // plain task-space control (the headline workload) runs an instantiation without the general kernel's spills
  if (osc_plain(p, N, c.frame, KD, c.tv != nullptr, c.ierr != nullptr)) return osc_launch<T, N, ORTHO, KD, true>(h, p, c);
  return osc_launch<T, N, ORTHO, KD, false>(h, p, c);
}

template <typename T>
void fill_rollout_args(const RolloutCall &c, RolloutArgs<T> &a) {
  a.q = static_cast<T *>(c.q);
  a.dq = static_cast<T *>(c.dq);
  a.target = static_cast<const T *>(c.target);
  a.q_traj = static_cast<T *>(c.q_traj);
  a.dq_traj = static_cast<T *>(c.dq_traj);
  a.u_traj = static_cast<T *>(c.u_traj);
  a.ierr = static_cast<T *>(c.ierr);
  a.B = c.B;
  a.target_stride = c.target_stride;
  a.steps = c.steps;
  a.dt = T(c.dt);
}

template <typename T, int N, bool ORTHO, int KD, bool PLAIN>
int rollout_path_launch(const ChainHost &h, const abrb_osc_params &p, const RolloutPathCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, c.frame, c.xoff, O);
  RolloutPathArgs<T> a;
  fill_rollout_args<T>(c, a);
  a.tv = static_cast<const T *>(c.tv);
  a.x_traj = static_cast<T *>(c.x_traj);
  a.cost = static_cast<T *>(c.cost);
  a.tv_stride = c.tv_stride;
  a.effort = T(c.effort_weight);
  const size_t smem = (size_t)kWarps * OscSmem<T, N, ORTHO, KD>::kElems * sizeof(T);
  auto kern = rollout_kernel<T, N, ORTHO, KD, PLAIN, RolloutPathArgs<T>>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, O, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO, int KD>
int rollout_path_go(const ChainHost &h, const abrb_osc_params &p, const RolloutPathCall &c) {
  // as in generate: a path velocity needs the general instantiation; a shared or per-trajectory path does not matter
  if (osc_plain(p, N, c.frame, KD, c.tv != nullptr, c.ierr != nullptr))
    return rollout_path_launch<T, N, ORTHO, KD, true>(h, p, c);
  return rollout_path_launch<T, N, ORTHO, KD, false>(h, p, c);
}

template <typename T, int N, bool ORTHO, int KD, bool PLAIN>
int rollout_launch(const ChainHost &h, const abrb_osc_params &p, const RolloutCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, c.frame, c.xoff, O);
  RolloutArgs<T> a;
  fill_rollout_args<T>(c, a);
  const size_t smem = (size_t)kWarps * OscSmem<T, N, ORTHO, KD>::kElems * sizeof(T);
  auto kern = rollout_kernel<T, N, ORTHO, KD, PLAIN, RolloutArgs<T>>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, O, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO, int KD>
int rollout_go(const ChainHost &h, const abrb_osc_params &p, const RolloutCall &c) {
  if (osc_plain(p, N, c.frame, KD, false, c.ierr != nullptr)) return rollout_launch<T, N, ORTHO, KD, true>(h, p, c);
  return rollout_launch<T, N, ORTHO, KD, false>(h, p, c);
}

template <typename T, int N, bool ORTHO>
int null_go(const ChainHost &h, const abrb_null_params &z, const NullCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  NullK<T, N> Z;
  fill_null<T, N>(z, Z);
  NullArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.u = static_cast<T *>(c.u);
  a.B = c.B;
  const size_t smem = (size_t)kWarps * kPitch * (N < kChunk ? N : kChunk) * sizeof(T);
  null_kernel<T, N, ORTHO><<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, Z, a);
  count_launch();
  return (int)cudaGetLastError();
}

inline bool needs_kd6(const abrb_osc_params &p) { return p.ctrlr_dof[3] || p.ctrlr_dof[4] || p.ctrlr_dof[5]; }

}  // namespace

template <typename T, int N, bool ORTHO>
int ctrl_go(const ChainHost &h, const CtrlCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  CtrlArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.target = static_cast<const T *>(c.target);
  a.tv = static_cast<const T *>(c.tv);
  a.u = static_cast<T *>(c.u);
  a.B = c.B;
  a.target_stride = c.target_stride;
  a.tv_stride = c.tv_stride;
  a.kind = c.kind;
  a.flag_a = c.flag_a;
  a.flag_b = c.flag_b;
  a.kp = T(c.kp);
  a.kv = T(c.kv);
  const size_t smem = (size_t)kWarps * kPitch * N * sizeof(T);
  ctrl_kernel<T, N, ORTHO><<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <>
int launch_rbd<ABRB_N>(const ChainHost &h, const RbdCall &c) {
  return c.f32 ? rbd_dispatch<float, ABRB_N>(h, c) : rbd_dispatch<double, ABRB_N>(h, c);
}

#define ABRB_OSC_DISPATCH(GO, ...)                                                              \
  do {                                                                                          \
    const bool k6 = needs_kd6(p);                                                               \
    if (c.f32) {                                                                                \
      if (h.ortho) return k6 ? GO<float, ABRB_N, true, 6>(__VA_ARGS__) : GO<float, ABRB_N, true, 3>(__VA_ARGS__);    \
      return k6 ? GO<float, ABRB_N, false, 6>(__VA_ARGS__) : GO<float, ABRB_N, false, 3>(__VA_ARGS__);               \
    }                                                                                           \
    if (h.ortho) return k6 ? GO<double, ABRB_N, true, 6>(__VA_ARGS__) : GO<double, ABRB_N, true, 3>(__VA_ARGS__);    \
    return k6 ? GO<double, ABRB_N, false, 6>(__VA_ARGS__) : GO<double, ABRB_N, false, 3>(__VA_ARGS__);               \
  } while (0)

template <>
int launch_osc<ABRB_N>(const ChainHost &h, const abrb_osc_params &p, const OscCall &c) {
  ABRB_OSC_DISPATCH(osc_go, h, p, c);
}

template <>
int launch_rollout<ABRB_N>(const ChainHost &h, const abrb_osc_params &p, const RolloutCall &c) {
  ABRB_OSC_DISPATCH(rollout_go, h, p, c);
}

template <>
int launch_rollout_path<ABRB_N>(const ChainHost &h, const abrb_osc_params &p, const RolloutPathCall &c) {
  ABRB_OSC_DISPATCH(rollout_path_go, h, p, c);
}

template <>
int launch_null<ABRB_N>(const ChainHost &h, const abrb_null_params &z, const NullCall &c) {
  if (c.f32) return h.ortho ? null_go<float, ABRB_N, true>(h, z, c) : null_go<float, ABRB_N, false>(h, z, c);
  return h.ortho ? null_go<double, ABRB_N, true>(h, z, c) : null_go<double, ABRB_N, false>(h, z, c);
}

template <typename T, int N, bool ORTHO>
int sliding_go(const ChainHost &h, const SlidingCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  SlidingArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.target = static_cast<const T *>(c.target);
  a.tv = static_cast<const T *>(c.tv);
  a.ta = static_cast<const T *>(c.ta);
  a.u = static_cast<T *>(c.u);
  a.s = static_cast<T *>(c.s);
  a.B = c.B;
  a.target_stride = c.target_stride;
  a.tv_stride = c.tv_stride;
  a.ta_stride = c.ta_stride;
  a.cartesian = c.cartesian;
  a.frame = c.frame;
  a.kd = T(c.kd);
  a.lamb = T(c.lamb);
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  const size_t smem = (size_t)kWarps * kPitch * N * sizeof(T);
  sliding_kernel<T, N, ORTHO><<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int ik_go(const ChainHost &h, const IkCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  IkArgs<T> a;
  a.position = static_cast<const T *>(c.position);
  a.target = static_cast<const T *>(c.target);
  a.pos_path = static_cast<T *>(c.pos_path);
  a.vel_path = static_cast<T *>(c.vel_path);
  a.B = c.B;
  a.target_stride = c.target_stride;
  a.steps = c.steps;
  a.method = c.method;
  a.max_dx = T(c.max_dx * c.dt);
  a.max_dr = T(c.max_dr * c.dt);
  a.max_dq = T(c.max_dq * c.dt);
  const size_t smem = (size_t)kWarps * kPitch * N * sizeof(T);
  ik_kernel<T, N, ORTHO><<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int plant_go(const ChainHost &h, const PlantCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  PlantArgs<T> a;
  a.q = static_cast<T *>(c.q);
  a.dq = static_cast<T *>(c.dq);
  a.u = static_cast<const T *>(c.u);
  a.path = static_cast<const T *>(c.path);
  a.q_traj = static_cast<T *>(c.q_traj);
  a.dq_traj = static_cast<T *>(c.dq_traj);
  a.u_traj = static_cast<T *>(c.u_traj);
  a.x_traj = static_cast<T *>(c.x_traj);
  a.cost = static_cast<T *>(c.cost);
  a.B = c.B;
  a.u_stride = c.u_stride;
  a.path_stride = c.path_stride;
  a.steps = c.steps;
  a.frame = c.frame;
  a.comp_g = c.compensate_gravity;
  a.dt = T(c.dt);
  a.effort = T(c.effort_weight);
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  const size_t smem = (size_t)kWarps * WarpSmem<T, N, ORTHO, (N > 3 ? N : 3)>::kElems * sizeof(T);
  auto kern = plant_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int dyn_go(const ChainHost &h, const DynCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  DynArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.in = static_cast<const T *>(c.in);
  a.out = static_cast<T *>(c.out);
  a.B = c.B;
  a.kind = c.kind;
  const size_t smem = (size_t)kWarps * WarpSmem<T, N, ORTHO, N>::kElems * sizeof(T);
  auto kern = dyn_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int regressor_go(const ChainHost &h, const RegressorCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  RegressorArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.ddq = static_cast<const T *>(c.ddq);
  a.Yt = static_cast<T *>(c.Yt);
  a.B = c.B;
  for (int i = 0; i < 6; ++i) a.gravity[i] = T(c.gravity[i]);
  const size_t smem = (size_t)kWarps * WarpSmem<T, N, ORTHO, RegressorLayout<N>::kHalf>::kElems * sizeof(T);
  auto kern = regressor_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <>
int launch_plant<ABRB_N>(const ChainHost &h, const PlantCall &c) {
  if (c.f32) return h.ortho ? plant_go<float, ABRB_N, true>(h, c) : plant_go<float, ABRB_N, false>(h, c);
  return h.ortho ? plant_go<double, ABRB_N, true>(h, c) : plant_go<double, ABRB_N, false>(h, c);
}

template <typename T, int N, bool ORTHO, int KIND>
int ctrl_rollout_go(const ChainHost &h, const CtrlRolloutCall &c) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  CtrlRolloutArgs<T> a;
  a.q = static_cast<T *>(c.q);
  a.dq = static_cast<T *>(c.dq);
  a.path = static_cast<const T *>(c.path);
  a.pv = static_cast<const T *>(c.pv);
  a.pa = static_cast<const T *>(c.pa);
  a.q_traj = static_cast<T *>(c.q_traj);
  a.dq_traj = static_cast<T *>(c.dq_traj);
  a.u_traj = static_cast<T *>(c.u_traj);
  a.x_traj = static_cast<T *>(c.x_traj);
  a.cost = static_cast<T *>(c.cost);
  a.B = c.B;
  a.path_stride = c.path_stride;
  a.pv_stride = c.pv_stride;
  a.pa_stride = c.pa_stride;
  a.steps = c.steps;
  a.frame = c.frame;
  a.G.kp = T(c.kp);
  a.G.kv = T(c.kv);
  a.G.kd = T(c.kd);
  a.G.lamb = T(c.lamb);
  a.G.gravity = c.gravity;
  a.G.cartesian = c.cartesian;
  a.dt = T(c.dt);
  a.effort = T(c.effort_weight);
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  const size_t smem = (size_t)kWarps * WarpSmem<T, N, ORTHO, (N > 3 ? N : 3)>::kElems * sizeof(T);
  auto kern = ctrl_rollout_kernel<T, N, ORTHO, KIND>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid_for(c.B, 8), kBlock, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int KIND>
int ctrl_rollout_ortho(const ChainHost &h, const CtrlRolloutCall &c) {
  return h.ortho ? ctrl_rollout_go<T, ABRB_N, true, KIND>(h, c) : ctrl_rollout_go<T, ABRB_N, false, KIND>(h, c);
}

template <>
int launch_ctrl_rollout<ABRB_N>(const ChainHost &h, const CtrlRolloutCall &c) {
  if (c.kind == kCtrlJoint)
    return c.f32 ? ctrl_rollout_ortho<float, kCtrlJoint>(h, c) : ctrl_rollout_ortho<double, kCtrlJoint>(h, c);
  return c.f32 ? ctrl_rollout_ortho<float, kCtrlSliding>(h, c) : ctrl_rollout_ortho<double, kCtrlSliding>(h, c);
}

template <>
int launch_dyn<ABRB_N>(const ChainHost &h, const DynCall &c) {
  if (c.f32) return h.ortho ? dyn_go<float, ABRB_N, true>(h, c) : dyn_go<float, ABRB_N, false>(h, c);
  return h.ortho ? dyn_go<double, ABRB_N, true>(h, c) : dyn_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_regressor<ABRB_N>(const ChainHost &h, const RegressorCall &c) {
  if (c.f32) return h.ortho ? regressor_go<float, ABRB_N, true>(h, c) : regressor_go<float, ABRB_N, false>(h, c);
  return h.ortho ? regressor_go<double, ABRB_N, true>(h, c) : regressor_go<double, ABRB_N, false>(h, c);
}

template <typename T, int N, bool ORTHO>
int dyn_jac_go(const ChainHost &h, const DynJacCall &c) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  DynJacArgs<T> a;
  a.q = static_cast<const T *>(c.q);
  a.dq = static_cast<const T *>(c.dq);
  a.in = static_cast<const T *>(c.in);
  a.d_q = static_cast<T *>(c.d_q);
  a.d_dq = static_cast<T *>(c.d_dq);
  a.d_in = static_cast<T *>(c.d_in);
  a.B = c.B;
  a.kind = c.kind;
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const size_t smem = DualSmem<T, N, ORTHO>::kBytes;
  auto kern = dyn_jac_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  const int64_t blocks = (c.B + kW - 1) / kW, cap = (int64_t)num_sms() * 16;
  kern<<<(unsigned)(blocks < cap ? blocks : cap), DualBlock<ORTHO>::value, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int plant_vjp_go(const ChainHost &h, const PlantVjpCall &c) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  PlantVjpArgs<T> a;
  a.q0 = static_cast<const T *>(c.q0);
  a.dq0 = static_cast<const T *>(c.dq0);
  a.u = static_cast<const T *>(c.u);
  a.path = static_cast<const T *>(c.path);
  a.q_traj = static_cast<const T *>(c.q_traj);
  a.dq_traj = static_cast<const T *>(c.dq_traj);
  a.g_cost = static_cast<const T *>(c.g_cost);
  a.g_q = static_cast<const T *>(c.g_q);
  a.g_dq = static_cast<const T *>(c.g_dq);
  a.g_q_traj = static_cast<const T *>(c.g_q_traj);
  a.g_dq_traj = static_cast<const T *>(c.g_dq_traj);
  a.g_u_traj = static_cast<const T *>(c.g_u_traj);
  a.g_x_traj = static_cast<const T *>(c.g_x_traj);
  a.gu = static_cast<T *>(c.gu);
  a.gq0 = static_cast<T *>(c.gq0);
  a.gdq0 = static_cast<T *>(c.gdq0);
  a.B = c.B;
  a.u_stride = c.u_stride;
  a.path_stride = c.path_stride;
  a.steps = c.steps;
  a.frame = c.frame;
  a.comp_g = c.compensate_gravity;
  a.dt = T(c.dt);
  a.effort = T(c.effort_weight);
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const size_t smem = DualSmem<T, N, ORTHO>::kBytes;
  auto kern = plant_vjp_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  const int64_t blocks = (c.B + kW - 1) / kW, cap = (int64_t)num_sms() * 16;
  kern<<<(unsigned)(blocks < cap ? blocks : cap), DualBlock<ORTHO>::value, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <typename T, int N, bool ORTHO>
int joint_vjp_go(const ChainHost &h, const JointVjpCall &c) {
  ChainK<Dual<T>, N> P;
  fill_chain<Dual<T>, N>(h, P);
  JointVjpArgs<T> a;
  a.q0 = static_cast<const T *>(c.q0);
  a.dq0 = static_cast<const T *>(c.dq0);
  a.path = static_cast<const T *>(c.path);
  a.pv = static_cast<const T *>(c.pv);
  a.q_traj = static_cast<const T *>(c.q_traj);
  a.dq_traj = static_cast<const T *>(c.dq_traj);
  a.g_cost = static_cast<const T *>(c.g_cost);
  a.g_q = static_cast<const T *>(c.g_q);
  a.g_dq = static_cast<const T *>(c.g_dq);
  a.g_q_traj = static_cast<const T *>(c.g_q_traj);
  a.g_dq_traj = static_cast<const T *>(c.g_dq_traj);
  a.g_u_traj = static_cast<const T *>(c.g_u_traj);
  a.g_x_traj = static_cast<const T *>(c.g_x_traj);
  a.g_path = static_cast<T *>(c.g_path);
  a.g_pv = static_cast<T *>(c.g_pv);
  a.g_gains = static_cast<T *>(c.g_gains);
  a.gq0 = static_cast<T *>(c.gq0);
  a.gdq0 = static_cast<T *>(c.gdq0);
  a.B = c.B;
  a.path_stride = c.path_stride;
  a.pv_stride = c.pv_stride;
  a.steps = c.steps;
  a.frame = c.frame;
  a.gravity = c.gravity;
  a.kp = T(c.kp);
  a.kv = T(c.kv);
  a.dt = T(c.dt);
  a.effort = T(c.effort_weight);
  for (int i = 0; i < 3; ++i) a.xoff[i] = c.xoff ? T(c.xoff[i]) : T(0);
  constexpr int kW = DualBlock<ORTHO>::value / 32;
  const size_t smem = JointDualSmem<T, N, ORTHO>::kBytes;
  auto kern = joint_vjp_kernel<T, N, ORTHO>;
  cudaError_t e = set_smem(kern, smem);
  if (e != cudaSuccess) return (int)e;
  const int64_t blocks = (c.B + kW - 1) / kW, cap = (int64_t)num_sms() * 16;
  kern<<<(unsigned)(blocks < cap ? blocks : cap), DualBlock<ORTHO>::value, smem, c.stream>>>(P, a);
  count_launch();
  return (int)cudaGetLastError();
}

template <>
int launch_joint_vjp<ABRB_N>(const ChainHost &h, const JointVjpCall &c) {
  if (c.f32) return h.ortho ? joint_vjp_go<float, ABRB_N, true>(h, c) : joint_vjp_go<float, ABRB_N, false>(h, c);
  return h.ortho ? joint_vjp_go<double, ABRB_N, true>(h, c) : joint_vjp_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_dyn_jac<ABRB_N>(const ChainHost &h, const DynJacCall &c) {
  if (c.f32) return h.ortho ? dyn_jac_go<float, ABRB_N, true>(h, c) : dyn_jac_go<float, ABRB_N, false>(h, c);
  return h.ortho ? dyn_jac_go<double, ABRB_N, true>(h, c) : dyn_jac_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_plant_vjp<ABRB_N>(const ChainHost &h, const PlantVjpCall &c) {
  if (c.f32) return h.ortho ? plant_vjp_go<float, ABRB_N, true>(h, c) : plant_vjp_go<float, ABRB_N, false>(h, c);
  return h.ortho ? plant_vjp_go<double, ABRB_N, true>(h, c) : plant_vjp_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_ik<ABRB_N>(const ChainHost &h, const IkCall &c) {
  if (c.f32) return h.ortho ? ik_go<float, ABRB_N, true>(h, c) : ik_go<float, ABRB_N, false>(h, c);
  return h.ortho ? ik_go<double, ABRB_N, true>(h, c) : ik_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_sliding<ABRB_N>(const ChainHost &h, const SlidingCall &c) {
  if (c.f32) return h.ortho ? sliding_go<float, ABRB_N, true>(h, c) : sliding_go<float, ABRB_N, false>(h, c);
  return h.ortho ? sliding_go<double, ABRB_N, true>(h, c) : sliding_go<double, ABRB_N, false>(h, c);
}

template <>
int launch_ctrl<ABRB_N>(const ChainHost &h, const CtrlCall &c) {
  if (c.f32) return h.ortho ? ctrl_go<float, ABRB_N, true>(h, c) : ctrl_go<float, ABRB_N, false>(h, c);
  return h.ortho ? ctrl_go<double, ABRB_N, true>(h, c) : ctrl_go<double, ABRB_N, false>(h, c);
}

#if ABRB_N == 1
// ------------------------------------------------------------------------------------------------ path planner
// Independent of the joint count, so only the ABRB_N == 1 unit compiles it.  Both phases evaluate the planner in fp64
// (abrb_path.cuh); phase 2 reads phase 1's record instead of repeating the search, so every row's length and segment
// split are phase 1's by construction.
namespace {

constexpr int kPathPlanBlock = 128;  // four rows per CTA, one warp each
constexpr int kPathBlock = 256;      // phase 2: one CTA per row

// path::HostSum's order on one warp: lane l sums elements lo + l, lo + l + 32, ... then an xor butterfly.
struct WarpSum {
  template <class F>
  __device__ double operator()(int lo, int n, F f) const {
    const int lane = threadIdx.x & 31;
    double acc = 0.0;
    for (int i = lo + lane; i < n; i += 32) acc += f(i);
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    return acc;
  }
};

__global__ void __launch_bounds__(kPathPlanBlock) path_plan_kernel(const PathCall c) {
  const int64_t b = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (b >= c.B) return;  // warp-uniform
  abrb_path_rec rec{0.0, 0, 0, 0, 0};
  const int64_t len =
      path::plan_row(c.p, c.table, c.start + 3 * b, c.target + 3 * b, c.max_v[b], c.v0[b], c.v1[b], rec, WarpSum{});
  if ((threadIdx.x & 31) == 0) {
    c.lengths[b] = len;
    c.plan[b] = rec;
  }
}

// Inclusive scan over the CTA (Hillis-Steele in each warp, then the warp totals in order).  Thread 0 gets its own x
// back unchanged.  wsum: kPathBlock / 32 doubles of shared memory.
__device__ double block_incl_scan(double x, double *wsum) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int off = 1; off < 32; off <<= 1) {
    const double y = __shfl_up_sync(0xffffffffu, x, off);
    if (lane >= off) x += y;
  }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (w > 0) {
    double pre = wsum[0];
    for (int k = 1; k < w; ++k) pre += wsum[k];
    x = pre + x;
  }
  __syncthreads();
  return x;
}

// phase 2 shared memory: arc[P], xyz[3P], path_steps window [kPathBlock + 2], warp sums [8], last row [12], p_0, p_end
__host__ __device__ constexpr size_t path_fill_smem(int P) {
  return sizeof(double) * (size_t(4) * P + kPathBlock + 2 + kPathBlock / 32 + 12 + 6);
}

template <typename T>
__global__ void __launch_bounds__(kPathBlock) path_fill_kernel(const PathCall c) {
  extern __shared__ double sm[];
  __shared__ double carry_sh;
  const int P = c.p.n_points, t = threadIdx.x;
  double *arc = sm, *xyz = arc + P, *ps = xyz + 3 * P, *wsum = ps + kPathBlock + 2, *last = wsum + kPathBlock / 32,
         *ends = last + 12;
  const int64_t b = blockIdx.x;
  const int w = c.so ? 12 : 6;
  T *out = static_cast<T *>(c.path);
  const int64_t len = c.lengths[b];
  const int64_t S = len < c.s_max ? len : c.s_max;
  if (S < 2) {  // a row the planner rejected: defined contents, never a path
    for (int64_t k = t; k < c.s_max; k += kPathBlock)
      for (int q = 0; q < w; ++q) out[(k * c.B + b) * w + q] = T(NAN);
    return;
  }
  path::Frame F;
  path::frame_of(c.start + 3 * b, c.target + 3 * b, F);
  // dist_steps = cumsum(curve_dist_steps) and warped_xyz, chunk by chunk
  double carry = 0.0;
  for (int i0 = 0; i0 < P; i0 += kPathBlock) {
    const int i = i0 + t;
    const double s = block_incl_scan((i > 0 && i < P) ? path::seg_len(F, c.table, i) : 0.0, wsum) + carry;
    if (i < P) {
      arc[i] = s;
      path::warp_point(F, c.table, i, xyz + 3 * i);
    }
    if (t == kPathBlock - 1) carry_sh = s;
    __syncthreads();
    carry = carry_sh;
    __syncthreads();
  }
  const path::Profile Pr = path::profile_of(c.p, c.plan[b], c.v0[b], c.v1[b]);
  // path_steps = cumsum(stacked * dt), one window of kPathBlock steps at a time.  Pass 0 finds p_0 and p_end (the
  // SLERP fraction needs them at every step); pass 1 writes the rows.  Both passes compute every path_steps value with
  // the same code, so p_end is the position of row S - 1.
  const int passes = w == 12 ? 2 : 1;
  double q0[4], q1[4];
  if (w == 12) {
    path::unit_quat(c.so + 3 * b, c.p.axes, q0);
    path::unit_quat(c.to + 3 * b, c.p.axes, q1);
  }
  for (int pass = 2 - passes; pass < 2; ++pass) {
    carry = 0.0;
    for (int64_t k0 = 0; k0 < S; k0 += kPathBlock) {
      const int64_t k = k0 + t;
      const double s = block_incl_scan(k < S ? path::step_at(Pr, int(k)) : 0.0, wsum) + carry;
      ps[t + 1] = s;
      if (t == 0) ps[0] = carry;
      if (t == kPathBlock - 1) ps[kPathBlock + 1] = k + 1 < S ? s + path::step_at(Pr, int(k + 1)) : 0.0;
      if (pass == 0) {
        if (k == 0) path::interp(arc, xyz, P, s, ends);
        if (k == S - 1) path::interp(arc, xyz, P, s, ends + 3);
      }
      __syncthreads();
      if (pass == 1 && k < S) {
        double p[3], pm[3] = {0, 0, 0}, pp[3] = {0, 0, 0}, r[12];
        path::interp(arc, xyz, P, s, p);
        if (k > 0) path::interp(arc, xyz, P, ps[t], pm);
        if (k < S - 1) path::interp(arc, xyz, P, ps[t + 2], pp);
        for (int q = 0; q < 3; ++q) {
          r[q] = p[q];
          r[3 + q] = path::gradient_at(pm[q], p[q], pp[q], int(k), int(S), c.p.dt);
        }
        if (w == 12) {
          double e[3], em[3] = {0, 0, 0}, ep[3] = {0, 0, 0};
          path::orient_at(q0, q1, c.p.axes, ends, ends + 3, p, e);
          if (k > 0) path::orient_at(q0, q1, c.p.axes, ends, ends + 3, pm, em);
          if (k < S - 1) path::orient_at(q0, q1, c.p.axes, ends, ends + 3, pp, ep);
          for (int q = 0; q < 3; ++q) {
            r[6 + q] = e[q];
            r[9 + q] = path::gradient_at(em[q], e[q], ep[q], int(k), int(S), c.p.dt);
          }
        }
        T *o = out + (k * c.B + b) * w;
        for (int q = 0; q < w; ++q) o[q] = T(r[q]);
        if (k == S - 1)
          for (int q = 0; q < w; ++q) last[q] = r[q];
      }
      carry = ps[kPathBlock];
      __syncthreads();
    }
  }
  // rows past the path repeat its last row (the reference's clamped next())
  for (int64_t k = S + t; k < c.s_max; k += kPathBlock) {
    T *o = out + (k * c.B + b) * w;
    for (int q = 0; q < w; ++q) o[q] = T(last[q]);
  }
}

}  // namespace

int launch_path_plan(const PathCall &c) {
  const int64_t grid = (c.B * 32 + kPathPlanBlock - 1) / kPathPlanBlock;
  path_plan_kernel<<<(unsigned)grid, kPathPlanBlock, 0, c.stream>>>(c);
  count_launch();
  return (int)cudaGetLastError();
}

int launch_path_fill(const PathCall &c) {
  const size_t smem = path_fill_smem(c.p.n_points);
  const void *fn = c.f32 ? (const void *)path_fill_kernel<float> : (const void *)path_fill_kernel<double>;
  if (smem > 48 * 1024) {
    const int e = (int)cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e) return e;
  }
  if (c.f32)
    path_fill_kernel<float><<<(unsigned)c.B, kPathBlock, smem, c.stream>>>(c);
  else
    path_fill_kernel<double><<<(unsigned)c.B, kPathBlock, smem, c.stream>>>(c);
  count_launch();
  return (int)cudaGetLastError();
}
#endif  // ABRB_N == 1

}  // namespace abrb
