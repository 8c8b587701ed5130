// api.cu — the C ABI of libabrb.so (include/abrb.h): handle management, argument checking, dispatch on the
// joint count to the per-N kernel translation units, host-pointer convenience variants.
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <utility>

#include "abrb_launch.hpp"

using namespace abrb;

struct abrb_model {
  abrb_chain_desc desc;
  ChainHost host;
};

struct abrb_osc {
  const abrb_model *model;
  abrb_osc_params params;
  int64_t host_chunk = 0;  // option "host_chunk_states": states per pipeline chunk of the *_host entry points, 0 = auto
  int host_streams = 2;    // option "host_upload_streams": copy streams per chunk (1: q, dq, target in turn; 2: dq beside
                           // q; 3: per-state targets on a stream of their own as well)
};

// Symmetric gather buffers of one rank (include/abrb.h): one cudaMalloc'd region [ n_buffers x bytes | flags | counter ]
// exported with CUDA IPC; `peer[r]` is rank r's region mapped into this process (own region for r == rank).
struct abrb_gather {
  int rank = 0, world = 1, n_buffers = 1, dev = 0;
  size_t bytes = 0;       // per buffer
  size_t flag_off = 0;    // byte offset of flags[kMaxPeers] (unsigned long long) in a region
  size_t counter_off = 0; // byte offset of the CTA counter + status word
  void *peer[kMaxPeers] = {nullptr};
  bool imported[kMaxPeers] = {false};
  unsigned long long epoch = 0;  // launches issued so far (ranks call in lockstep, so epochs agree)
};

namespace {

thread_local std::string g_err;
std::atomic<int64_t> g_launches{0};

int fail(int code, const std::string &msg) {
  g_err = msg;
  return code;
}

int cuda_fail(int e, const char *where) {
  return fail(ABRB_ECUDA, std::string(where) + ": " + cudaGetErrorString((cudaError_t)e));
}

// the joint counts kernels.cu is compiled for (Makefile JOINTS)
#define ABRB_EACH_N(X) X(1) X(2) X(3) X(4) X(5) X(6) X(7)

bool n_supported(int n) {
#define X(k) if (n == k) return true;
  ABRB_EACH_N(X)
#undef X
  return false;
}

int ensure_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return fail(ABRB_ECUDA, "no CUDA device available (libabrb has no CPU fallback)");
  }
  return ABRB_OK;
}

// The kernels read and write with scalar (element-sized) accesses only, so element alignment is all they need: a
// row slice of a contiguous (B, n) array (q[1:], a rank's shard at an odd row) is a valid argument.
bool aligned_elem(const void *p, bool f32) { return (reinterpret_cast<uintptr_t>(p) & (f32 ? 3u : 7u)) == 0; }

// grow-only device workspace for the *_host entry points (one per host thread).  The OSC host path has kSlots
// independent pipeline slots (own device region, own streams) so that consecutive asynchronous calls overlap:
// slot 1's H2D runs under slot 0's kernel and D2H (PCIe is full duplex, and the copy engines run beside the SMs).
constexpr int kSlots = 2, kLanes = 2;
struct Workspace {
  void *ptr = nullptr;
  size_t cap = 0;
  int dev = -1;
  cudaStream_t stream = nullptr;
  struct Slot {
    void *ptr = nullptr;
    size_t cap = 0;
    cudaStream_t lanes[kLanes] = {nullptr, nullptr};  // chunk pipeline inside one call
    cudaStream_t side[kLanes] = {nullptr, nullptr};   // second copy stream of each lane (dq goes up beside q)
    cudaEvent_t side_done[kLanes] = {nullptr, nullptr};
    cudaStream_t side2[kLanes] = {nullptr, nullptr};  // third copy stream of each lane (per-state targets)
    cudaEvent_t side2_done[kLanes] = {nullptr, nullptr};
    int used = 0;                                      // lanes with work in flight
  } slots[kSlots];
  void release() {
    if (dev < 0) return;
    int cur = 0;
    if (cudaGetDevice(&cur) != cudaSuccess) return;  // process is shutting down
    cudaSetDevice(dev);
    cudaFree(ptr);
    if (stream) cudaStreamDestroy(stream);
    for (auto &sl : slots) {
      cudaFree(sl.ptr);
      for (int l = 0; l < kLanes; ++l) {
        if (sl.lanes[l]) cudaStreamDestroy(sl.lanes[l]);
        if (sl.side[l]) cudaStreamDestroy(sl.side[l]);
        if (sl.side_done[l]) cudaEventDestroy(sl.side_done[l]);
        if (sl.side2[l]) cudaStreamDestroy(sl.side2[l]);
        if (sl.side2_done[l]) cudaEventDestroy(sl.side2_done[l]);
      }
      sl = Slot();
    }
    cudaSetDevice(cur);
    ptr = nullptr;
    cap = 0;
    stream = nullptr;
    dev = -1;
  }
  ~Workspace() { release(); }
  int bind() {  // make the workspace belong to the calling thread's current device
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e != cudaSuccess) return (int)e;
    if (dev != cur) {  // the thread switched devices: streams and memory belong to the device they were made on
      release();
      dev = cur;
    }
    if (stream == nullptr) {
      e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
      if (e != cudaSuccess) return (int)e;
      for (auto &sl : slots)
        for (int l = 0; l < kLanes; ++l) {
          e = cudaStreamCreateWithFlags(&sl.lanes[l], cudaStreamNonBlocking);
          if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&sl.side[l], cudaStreamNonBlocking);
          if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.side_done[l], cudaEventDisableTiming);
          if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&sl.side2[l], cudaStreamNonBlocking);
          if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.side2_done[l], cudaEventDisableTiming);
          if (e != cudaSuccess) return (int)e;
        }
    }
    return 0;
  }
  int ensure(size_t bytes) {
    int e = bind();
    if (e) return e;
    if (bytes <= cap) return 0;
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
    cudaError_t ce = cudaMalloc(&ptr, bytes);
    if (ce != cudaSuccess) return (int)ce;
    cap = bytes;
    return 0;
  }
  int ensure_slot(int i, size_t bytes) {
    int e = bind();
    if (e) return e;
    Slot &sl = slots[i];
    if (bytes <= sl.cap) return 0;
    if (sl.ptr) cudaFree(sl.ptr);  // synchronises with anything still using it
    sl.ptr = nullptr;
    sl.cap = 0;
    cudaError_t ce = cudaMalloc(&sl.ptr, bytes);
    if (ce != cudaSuccess) return (int)ce;
    sl.cap = bytes;
    return 0;
  }
  int wait_slot(int i) {  // returns the first CUDA error of the slot's lanes
    Slot &sl = slots[i];
    cudaError_t first = cudaSuccess;
    for (int l = 0; l < sl.used; ++l) {
      cudaError_t e = cudaStreamSynchronize(sl.side[l]);
      if (e != cudaSuccess && first == cudaSuccess) first = e;
      e = cudaStreamSynchronize(sl.side2[l]);
      if (e != cudaSuccess && first == cudaSuccess) first = e;
      e = cudaStreamSynchronize(sl.lanes[l]);
      if (e != cudaSuccess && first == cudaSuccess) first = e;
    }
    sl.used = 0;
    return (int)first;
  }
};
thread_local Workspace g_ws;

size_t align_up(size_t v) { return (v + 255) & ~size_t(255); }

// Tile counters of the OSC kernel's dynamic tile scheduling: every launch takes the next of kSchedSlots {next tile, CTAs
// done} pairs of its device (zeroed once; the launch's last CTA re-arms its pair).  Launches on one stream are ordered,
// so a pair can only be shared by two launches in flight if 4096 launches were enqueued between them on other streams.
// Allocated at the first launch per device (not inside a CUDA-graph capture) and kept for the life of the process.
constexpr int kSchedSlots = 4096, kMaxDevices = 64;
struct SchedPool {
  int *base = nullptr;
  bool failed = false;
  std::atomic<unsigned> seq{0};
};
SchedPool g_sched[kMaxDevices];
std::mutex g_sched_mu;

int *sched_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  SchedPool &p = g_sched[dev];
  if (p.base == nullptr) {
    std::lock_guard<std::mutex> lock(g_sched_mu);
    if (p.base == nullptr && !p.failed) {
      int *b = nullptr;
      if (cudaMalloc(&b, kSchedSlots * 2 * sizeof(int)) == cudaSuccess &&
          cudaMemset(b, 0, kSchedSlots * 2 * sizeof(int)) == cudaSuccess) {
        p.base = b;
      } else {
        cudaGetLastError();
        p.failed = true;  // static tile assignment from now on
      }
    }
  }
  if (p.base == nullptr) return nullptr;
  return p.base + 2 * (p.seq.fetch_add(1, std::memory_order_relaxed) % kSchedSlots);
}

// a cudaMemcpyAsync that is rejected (bad pointer, wrong direction) fails at the call, NOT at the later synchronise
#define ABRB_CU(call, where)                                \
  do {                                                      \
    cudaError_t e_ = (call);                                \
    if (e_ != cudaSuccess) return cuda_fail((int)e_, where); \
  } while (0)

// Consumer side of the fused all-gather: one thread per rank spins (system-scope acquire loads) until that rank has
// published `epoch` in our flag array, i.e. all its rows of this launch have landed in our buffer.
__global__ void gather_wait_kernel(const unsigned long long *flags, int world, unsigned long long epoch, int *status) {
  const int r = threadIdx.x;
  // launched as a programmatic dependent of the stream's previous kernel (the OSC kernel that feeds the gather): the
  // thread block is already resident when that kernel completes instead of paying a launch after it
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (r < world) {
    const long long t0 = clock64();
    for (;;) {
      unsigned long long v;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flags + r) : "memory");
      if (v >= epoch) break;
      if (clock64() - t0 > (6LL << 30)) {  // ~3 s: a peer never arrived; report instead of hanging the GPU
        *status = 1;
        break;
      }
      __nanosleep(100);
    }
  }
}

}  // namespace

namespace abrb {
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace abrb

extern "C" {

int abrb_version(void) { return ABRB_VERSION; }
const char *abrb_last_error(void) { return g_err.c_str(); }
int64_t abrb_launch_count(void) { return g_launches.load(); }

int abrb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return fail(ABRB_ECUDA, "cudaGetDeviceCount failed");
  }
  return n;
}

int abrb_model_create(const abrb_chain_desc *desc, abrb_model **out) {
  if (!desc || !out) return fail(ABRB_EINVAL, "abrb_model_create: NULL argument");
  *out = nullptr;
  if (desc->n_joints < 1 || desc->n_joints > ABRB_MAX_JOINTS || !n_supported(desc->n_joints))
    return fail(ABRB_ESHAPE, "abrb_model_create: n_joints not supported by this build");
  abrb_model *m = new (std::nothrow) abrb_model;
  if (!m) return fail(ABRB_ENOMEM, "abrb_model_create: out of memory");
  m->desc = *desc;
  std::string e = chain_from_desc(*desc, m->host);
  if (!e.empty()) {
    delete m;
    return fail(ABRB_ESHAPE, "abrb_model_create: " + e);
  }
  *out = m;
  return ABRB_OK;
}

int abrb_model_destroy(abrb_model *m) {
  delete m;
  return ABRB_OK;
}

int abrb_model_n_joints(const abrb_model *m) { return m ? m->host.n : fail(ABRB_EINVAL, "NULL model"); }
int abrb_model_is_orthonormal(const abrb_model *m) { return m ? (m->host.ortho ? 1 : 0) : fail(ABRB_EINVAL, "NULL model"); }

int abrb_frame_id(const abrb_model *m, const char *name) {
  if (!m) return fail(ABRB_EINVAL, "NULL model");
  int id = parse_frame(m->host.n, name);
  if (id < 0) return fail(ABRB_EFRAME, std::string("Invalid transformation name: ") + (name ? name : "(null)"));
  return id;
}

// ------------------------------------------------------------------------------------------------ rbd
static int rbd_eval(const abrb_model *m, int frame_id, const double *x_off, const void *q, const void *dq,
                    int64_t B, const abrb_rbd_out *out, void *stream, bool f32) {
  if (!m || !out) return fail(ABRB_EINVAL, "abrb_rbd_eval: NULL model/out");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_rbd_eval: B < 0");
  const int n = m->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, "abrb_rbd_eval: invalid frame id");
  if ((out->dJ || out->C) && !dq) return fail(ABRB_EINVAL, "abrb_rbd_eval: dJ / C need dq");
  if (B == 0) return ABRB_OK;
  if (!q) return fail(ABRB_EINVAL, "abrb_rbd_eval: NULL q");
  const void *ptrs[] = {q, dq, out->Tx, out->T, out->R, out->T_inv, out->quat, out->J, out->dJ, out->M, out->g, out->C};
  for (const void *p : ptrs)
    if (p && !aligned_elem(p, f32)) return fail(ABRB_EINVAL, "abrb_rbd_eval: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  RbdCall c{frame_id, x_off, q, dq, B, *out, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(k) case k: e = launch_rbd<k>(m->host, c); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, "abrb_rbd_eval") : ABRB_OK;
}

int abrb_rbd_eval_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q, const double *dq,
                      int64_t B, const abrb_rbd_out *out, void *stream) {
  return rbd_eval(m, frame_id, x_off, q, dq, B, out, stream, false);
}
int abrb_rbd_eval_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q, const float *dq,
                      int64_t B, const abrb_rbd_out *out, void *stream) {
  return rbd_eval(m, frame_id, x_off, q, dq, B, out, stream, true);
}

static int rbd_eval_host(const abrb_model *m, int frame_id, const double *x_off, const void *q, const void *dq,
                         int64_t B, const abrb_rbd_out *out, bool f32) {
  if (!m || !out) return fail(ABRB_EINVAL, "abrb_rbd_eval_host: NULL model/out");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_rbd_eval_host: B < 0");
  if (B == 0) return ABRB_OK;
  if (!q) return fail(ABRB_EINVAL, "abrb_rbd_eval_host: NULL q");
  int rc = ensure_device();
  if (rc) return rc;
  const size_t es = f32 ? 4 : 8, n = (size_t)m->host.n;
  const size_t len[10] = {3, 16, 9, 16, 4, 6 * n, 6 * n, n * n, n, n * n};
  void *const host_out[10] = {out->Tx, out->T, out->R, out->T_inv, out->quat, out->J, out->dJ, out->M, out->g, out->C};
  size_t total = 2 * align_up((size_t)B * n * es);
  for (int i = 0; i < 10; ++i)
    if (host_out[i]) total += align_up((size_t)B * len[i] * es);
  int e = g_ws.ensure(total);
  if (e) return cuda_fail(e, "abrb_rbd_eval_host(workspace)");
  char *base = static_cast<char *>(g_ws.ptr);
  size_t off = 0;
  auto take = [&](size_t bytes) { char *p = base + off; off += align_up(bytes); return (void *)p; };
  void *dq_q = take((size_t)B * n * es), *dq_dq = take((size_t)B * n * es);
  cudaStream_t s = g_ws.stream;
  ABRB_CU(cudaMemcpyAsync(dq_q, q, (size_t)B * n * es, cudaMemcpyHostToDevice, s), "abrb_rbd_eval_host(q)");
  if (dq) ABRB_CU(cudaMemcpyAsync(dq_dq, dq, (size_t)B * n * es, cudaMemcpyHostToDevice, s), "abrb_rbd_eval_host(dq)");
  void *dev_out[10];
  for (int i = 0; i < 10; ++i) dev_out[i] = host_out[i] ? take((size_t)B * len[i] * es) : nullptr;
  abrb_rbd_out d{dev_out[0], dev_out[1], dev_out[2], dev_out[3], dev_out[4], dev_out[5], dev_out[6], dev_out[7], dev_out[8], dev_out[9]};
  rc = rbd_eval(m, frame_id, x_off, dq_q, dq ? dq_dq : nullptr, B, &d, s, f32);
  if (rc) return rc;
  for (int i = 0; i < 10; ++i)
    if (host_out[i])
      ABRB_CU(cudaMemcpyAsync(host_out[i], dev_out[i], (size_t)B * len[i] * es, cudaMemcpyDeviceToHost, s),
              "abrb_rbd_eval_host(result)");
  cudaError_t ce = cudaStreamSynchronize(s);
  return ce ? cuda_fail(ce, "abrb_rbd_eval_host") : ABRB_OK;
}

int abrb_rbd_eval_host_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q, const double *dq,
                           int64_t B, const abrb_rbd_out *out) {
  return rbd_eval_host(m, frame_id, x_off, q, dq, B, out, false);
}
int abrb_rbd_eval_host_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q, const float *dq,
                           int64_t B, const abrb_rbd_out *out) {
  return rbd_eval_host(m, frame_id, x_off, q, dq, B, out, true);
}

// ------------------------------------------------------------------------------------------------ osc
int abrb_osc_create(const abrb_model *m, const abrb_osc_params *p, abrb_osc **out) {
  if (!m || !p || !out) return fail(ABRB_EINVAL, "abrb_osc_create: NULL argument");
  *out = nullptr;
  std::string e = check_osc(m->host.n, *p);
  if (!e.empty()) return fail(ABRB_EUNSUP, "abrb_osc_create: " + e);
  abrb_osc *c = new (std::nothrow) abrb_osc;
  if (!c) return fail(ABRB_ENOMEM, "abrb_osc_create: out of memory");
  c->model = m;
  c->params = *p;
  if (const char *v = std::getenv("ABRB_HOST_CHUNK")) c->host_chunk = (int64_t)std::atoll(v);
  if (const char *v = std::getenv("ABRB_HOST_STREAMS")) {
    const int k = std::atoi(v);
    if (k >= 1 && k <= 3) c->host_streams = k;
  }
  *out = c;
  return ABRB_OK;
}

int abrb_osc_set_option(abrb_osc *c, const char *name, double value) {
  if (!c || !name) return fail(ABRB_EINVAL, "abrb_osc_set_option: NULL argument");
  if (std::strcmp(name, "host_chunk_states") == 0) {
    c->host_chunk = value > 0 ? (int64_t)value : 0;
    return ABRB_OK;
  }
  if (std::strcmp(name, "host_upload_streams") == 0) {
    if (!(value >= 1 && value <= 3)) return fail(ABRB_EINVAL, "abrb_osc_set_option: host_upload_streams must be 1, 2 or 3");
    c->host_streams = (int)value;
    return ABRB_OK;
  }
  return fail(ABRB_EINVAL, std::string("abrb_osc_set_option: unknown option ") + name);
}

int abrb_osc_destroy(abrb_osc *c) {
  delete c;
  return ABRB_OK;
}

static int osc_generate(const abrb_osc *c, int frame_id, const double *x_off, const void *q, const void *dq,
                        const void *target, int target_stride, const void *tv, int tv_stride, void *u, void *train,
                        void *ierr, int64_t B, void *stream, bool f32, const GatherArgs *gather = nullptr) {
  if (!c) return fail(ABRB_EINVAL, "abrb_osc_generate: NULL controller");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_osc_generate: B < 0");
  const int n = c->model->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, "abrb_osc_generate: invalid frame id");
  if ((target_stride != 0 && target_stride != 6) || (tv && tv_stride != 0 && tv_stride != 6))
    return fail(ABRB_EINVAL, "abrb_osc_generate: stride must be 0 (broadcast) or 6");
  if ((c->params.ki != 0.0) != (ierr != nullptr))
    return fail(ABRB_EINVAL, "abrb_osc_generate: integrated_error must be given if and only if ki != 0");
  if (B == 0) return ABRB_OK;
  if (!q || !dq || !target || (!u && !gather)) return fail(ABRB_EINVAL, "abrb_osc_generate: NULL q/dq/target/u");
  const void *ptrs[] = {q, dq, target, tv, u, train, ierr};
  for (const void *p : ptrs)
    if (p && !aligned_elem(p, f32)) return fail(ABRB_EINVAL, "abrb_osc_generate: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  OscCall k{frame_id, x_off, q, dq, target, tv, target_stride, tv_stride, u, train, B, f32, (cudaStream_t)stream};
  k.ierr = ierr;
  k.gather = gather;
  k.sched = sched_slot();
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_osc<j>(c->model->host, c->params, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, "abrb_osc_generate") : ABRB_OK;
}

int abrb_osc_generate_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q, const double *dq,
                          const double *target, int target_stride, const double *target_velocity, int tv_stride,
                          double *u, double *training_signal, double *integrated_error, int64_t B, void *stream) {
  return osc_generate(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                      training_signal, integrated_error, B, stream, false);
}
int abrb_osc_generate_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q, const float *dq,
                          const float *target, int target_stride, const float *target_velocity, int tv_stride,
                          float *u, float *training_signal, float *integrated_error, int64_t B, void *stream) {
  return osc_generate(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                      training_signal, integrated_error, B, stream, true);
}

// Host-pointer path.  One call = a chunked pipeline on the slot's two streams: every chunk carries its own H2D copies,
// its kernel launch and its D2H copies on ONE stream, consecutive chunks alternate streams, so chunk k+1's H2D overlaps
// chunk k's kernel and D2H.  The call returns as soon as everything is enqueued; abrb_osc_host_wait() (or the
// synchronous wrappers below) waits for the slot.  Every chunk costs copy and launch overheads of its own, so a
// blocking call uses two chunks up to ~200 k states and four above (tools/dbg/e2e_probe.py times the alternatives).
static int osc_generate_host_async(const abrb_osc *c, int frame_id, const double *x_off, const void *q, const void *dq,
                                   const void *target, int target_stride, const void *tv, int tv_stride, void *u,
                                   void *train, void *ierr, int64_t B, int slot, bool f32, bool blocking) {
  if (!c) return fail(ABRB_EINVAL, "abrb_osc_generate_host: NULL controller");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_osc_generate_host: B < 0");
  if (slot < 0 || slot >= kSlots) return fail(ABRB_EINVAL, "abrb_osc_generate_host: slot must be 0 or 1");
  if ((c->params.ki != 0.0) != (ierr != nullptr))
    return fail(ABRB_EINVAL, "abrb_osc_generate_host: integrated_error must be given if and only if ki != 0");
  if (B == 0) return ABRB_OK;
  if (!q || !dq || !target || !u) return fail(ABRB_EINVAL, "abrb_osc_generate_host: NULL q/dq/target/u");
  int rc = ensure_device();
  if (rc) return rc;
  int e = g_ws.bind();
  if (e) return cuda_fail(e, "abrb_osc_generate_host(workspace)");
  e = g_ws.wait_slot(slot);  // a slot is reused only after its previous batch has left it
  if (e) return cuda_fail(e, "abrb_osc_generate_host(previous batch of this slot)");
  const size_t es = f32 ? 4 : 8, n = (size_t)c->model->host.n;
  const size_t sz_state = (size_t)B * n * es, sz_six = (size_t)B * 6 * es;
  const size_t sz_t = target_stride ? sz_six : 6 * es, sz_tv = tv ? (tv_stride ? sz_six : 6 * es) : 0;
  e = g_ws.ensure_slot(slot, 4 * align_up(sz_state) + align_up(sz_t) + align_up(sz_tv) + (ierr ? align_up(sz_six) : 0) + 256);
  if (e) return cuda_fail(e, "abrb_osc_generate_host(workspace)");
  Workspace::Slot &sl = g_ws.slots[slot];
  char *base = static_cast<char *>(sl.ptr);
  size_t off = 0;
  auto take = [&](size_t bytes) { char *p = base + off; off += align_up(bytes); return (void *)p; };
  void *d_q = take(sz_state), *d_dq = take(sz_state), *d_u = take(sz_state), *d_tr = take(sz_state);
  void *d_t = take(sz_t), *d_tv = tv ? take(sz_tv) : nullptr, *d_ie = ierr ? take(sz_six) : nullptr;
  const size_t row = n * es;
  // Chunking inside one call pays when the caller then waits for the result (upload of chunk 1 under the kernel of chunk
  // 0).  A caller of the asynchronous entry points overlaps whole CALLS on the two slots,
  // and there the extra copies and launches of a chunked call only cost (tools/dbg/e2e_ab.py compares the two): one
  // chunk up to 196 608 states.
  int64_t chunk = (B < 49152 || (!blocking && B <= 196608))
                      ? B : ((B + (B <= 196608 ? 1 : 3)) / (B <= 196608 ? 2 : 4) + 127) / 128 * 128;
  if (c->host_chunk > 0) chunk = (c->host_chunk < B ? c->host_chunk : B + 127) / 128 * 128;
  if (chunk <= 0) chunk = B;
  const int n_chunks = (int)((B + chunk - 1) / chunk);
  sl.used = n_chunks < kLanes ? n_chunks : kLanes;
  // any failure below leaves copies in flight into the caller's buffers: drain the slot before reporting it
  auto bail = [&](int code) {
    g_ws.wait_slot(slot);
    return code;
  };
#define ABRB_CUH(call, where)                                    \
  do {                                                            \
    cudaError_t e_ = (call);                                      \
    if (e_ != cudaSuccess) return bail(cuda_fail((int)e_, where)); \
  } while (0)
  const char *where = "abrb_osc_generate_host(copy in)";
  if (!target_stride || (tv && !tv_stride)) {
    // broadcast rows go first on lane 0; the other lane waits for just these two small copies (the event is recorded
    // before chunk 0's own copies are enqueued, so the chunks still overlap)
    if (!target_stride) ABRB_CUH(cudaMemcpyAsync(d_t, target, sz_t, cudaMemcpyHostToDevice, sl.lanes[0]), where);
    if (tv && !tv_stride) ABRB_CUH(cudaMemcpyAsync(d_tv, tv, sz_tv, cudaMemcpyHostToDevice, sl.lanes[0]), where);
    if (sl.used > 1) {
      cudaEvent_t ev;
      ABRB_CUH(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), where);
      cudaError_t e1 = cudaEventRecord(ev, sl.lanes[0]);
      for (int l = 1; l < sl.used && e1 == cudaSuccess; ++l) e1 = cudaStreamWaitEvent(sl.lanes[l], ev, 0);
      cudaEventDestroy(ev);  // released once the recorded work has completed
      if (e1 != cudaSuccess) return bail(cuda_fail((int)e1, where));
    }
  }
  int lane = 0;
  for (int64_t b0 = 0; b0 < B; b0 += chunk, lane = (lane + 1) % kLanes) {
    const int64_t nb = B - b0 < chunk ? B - b0 : chunk;
    cudaStream_t s = sl.lanes[lane];
    const size_t off_s = (size_t)b0 * row, off_t = (size_t)b0 * 6 * es;
    auto at = [](const void *p, size_t o) { return (const void *)((const char *)p + o); };
    auto atw = [](void *p, size_t o) { return (void *)((char *)p + o); };
    // q, dq and the per-state targets go up on up to three streams at once (on some hosts one host->device stream
    // alone reaches less than half of what the link gives); the lane's stream waits
    // for the side copies before the kernel.  c->host_streams: 1, 2 (default) or 3.
    cudaStream_t s_dq = c->host_streams >= 2 ? sl.side[lane] : s;
    cudaStream_t s_t = c->host_streams >= 3 ? sl.side2[lane] : s;
    ABRB_CUH(cudaMemcpyAsync(atw(d_dq, off_s), at(dq, off_s), (size_t)nb * row, cudaMemcpyHostToDevice, s_dq), where);
    if (s_dq != s) ABRB_CUH(cudaEventRecord(sl.side_done[lane], s_dq), where);
    if (target_stride) {
      ABRB_CUH(cudaMemcpyAsync(atw(d_t, off_t), at(target, off_t), (size_t)nb * 6 * es, cudaMemcpyHostToDevice, s_t), where);
      if (s_t != s) ABRB_CUH(cudaEventRecord(sl.side2_done[lane], s_t), where);
    }
    ABRB_CUH(cudaMemcpyAsync(atw(d_q, off_s), at(q, off_s), (size_t)nb * row, cudaMemcpyHostToDevice, s), where);
    if (tv && tv_stride)
      ABRB_CUH(cudaMemcpyAsync(atw(d_tv, off_t), at(tv, off_t), (size_t)nb * 6 * es, cudaMemcpyHostToDevice, s), where);
    if (ierr)
      ABRB_CUH(cudaMemcpyAsync(atw(d_ie, off_t), at(ierr, off_t), (size_t)nb * 6 * es, cudaMemcpyHostToDevice, s), where);
    if (s_dq != s) ABRB_CUH(cudaStreamWaitEvent(s, sl.side_done[lane], 0), where);
    if (target_stride && s_t != s) ABRB_CUH(cudaStreamWaitEvent(s, sl.side2_done[lane], 0), where);
    rc = osc_generate(c, frame_id, x_off, at(d_q, off_s), at(d_dq, off_s), target_stride ? at(d_t, off_t) : d_t,
                      target_stride, tv ? (tv_stride ? at(d_tv, off_t) : d_tv) : nullptr, tv_stride, atw(d_u, off_s),
                      train ? atw(d_tr, off_s) : nullptr, ierr ? atw(d_ie, off_t) : nullptr, nb, s, f32);
    if (rc) return bail(rc);
    ABRB_CUH(cudaMemcpyAsync(atw(u, off_s), at(d_u, off_s), (size_t)nb * row, cudaMemcpyDeviceToHost, s),
             "abrb_osc_generate_host(result)");
    if (train)
      ABRB_CUH(cudaMemcpyAsync(atw(train, off_s), at(d_tr, off_s), (size_t)nb * row, cudaMemcpyDeviceToHost, s),
               "abrb_osc_generate_host(training signal)");
    if (ierr)
      ABRB_CUH(cudaMemcpyAsync(atw(ierr, off_t), at(d_ie, off_t), (size_t)nb * 6 * es, cudaMemcpyDeviceToHost, s),
               "abrb_osc_generate_host(integrated error)");
  }
#undef ABRB_CUH
  return ABRB_OK;
}

int abrb_osc_host_wait(const abrb_osc *c, int slot) {
  if (!c) return fail(ABRB_EINVAL, "abrb_osc_host_wait: NULL controller");
  if (slot < 0 || slot >= kSlots) return fail(ABRB_EINVAL, "abrb_osc_host_wait: slot must be 0 or 1");
  if (g_ws.dev < 0) return ABRB_OK;  // nothing was ever enqueued from this thread
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != g_ws.dev) cudaSetDevice(g_ws.dev);
  const int e = g_ws.wait_slot(slot);
  if (cur != g_ws.dev) cudaSetDevice(cur);
  return e ? cuda_fail(e, "abrb_osc_host_wait") : ABRB_OK;
}

int abrb_osc_generate_host_async_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q,
                                     const double *dq, const double *target, int target_stride,
                                     const double *target_velocity, int tv_stride, double *u, double *training_signal,
                                     double *integrated_error, int64_t B, int slot) {
  return osc_generate_host_async(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                                 training_signal, integrated_error, B, slot, false, false);
}
int abrb_osc_generate_host_async_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q,
                                     const float *dq, const float *target, int target_stride,
                                     const float *target_velocity, int tv_stride, float *u, float *training_signal,
                                     float *integrated_error, int64_t B, int slot) {
  return osc_generate_host_async(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                                 training_signal, integrated_error, B, slot, true, false);
}
int abrb_osc_generate_host_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q, const double *dq,
                               const double *target, int target_stride, const double *target_velocity,
                               int tv_stride, double *u, double *training_signal, double *integrated_error,
                               int64_t B) {
  const int rc = osc_generate_host_async(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride,
                                         u, training_signal, integrated_error, B, 0, false, true);
  return rc ? rc : abrb_osc_host_wait(c, 0);
}
int abrb_osc_generate_host_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q, const float *dq,
                               const float *target, int target_stride, const float *target_velocity, int tv_stride,
                               float *u, float *training_signal, float *integrated_error, int64_t B) {
  const int rc = osc_generate_host_async(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride,
                                         u, training_signal, integrated_error, B, 0, true, true);
  return rc ? rc : abrb_osc_host_wait(c, 0);
}

// ------------------------------------------------------------------------------------------------ peer gather
int abrb_gather_create(int rank, int world, int64_t bytes_per_buffer, int n_buffers, abrb_gather **out) {
  if (!out) return fail(ABRB_EINVAL, "abrb_gather_create: NULL argument");
  *out = nullptr;
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world || bytes_per_buffer <= 0 || n_buffers < 1 || n_buffers > 8)
    return fail(ABRB_EINVAL, "abrb_gather_create: need 0 <= rank < world <= 8, bytes > 0, 1 <= n_buffers <= 8");
  int rc = ensure_device();
  if (rc) return rc;
  abrb_gather *g = new (std::nothrow) abrb_gather;
  if (!g) return fail(ABRB_ENOMEM, "abrb_gather_create: out of memory");
  g->rank = rank;
  g->world = world;
  g->n_buffers = n_buffers;
  g->bytes = align_up((size_t)bytes_per_buffer);
  g->flag_off = g->bytes * (size_t)n_buffers;
  g->counter_off = g->flag_off + align_up(kMaxPeers * sizeof(unsigned long long));
  cudaGetDevice(&g->dev);
  const size_t total = g->counter_off + 256;
  cudaError_t e = cudaMalloc(&g->peer[rank], total);
  if (e == cudaSuccess) e = cudaMemset(static_cast<char *>(g->peer[rank]) + g->flag_off, 0, total - g->flag_off);
  if (e != cudaSuccess) {
    cudaFree(g->peer[rank]);
    delete g;
    return cuda_fail((int)e, "abrb_gather_create");
  }
  *out = g;
  return ABRB_OK;
}

int abrb_gather_export(const abrb_gather *g, unsigned char handle[64]) {
  if (!g || !handle) return fail(ABRB_EINVAL, "abrb_gather_export: NULL argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, g->peer[g->rank]);
  if (e != cudaSuccess) return cuda_fail((int)e, "abrb_gather_export");
  std::memcpy(handle, &h, 64);
  return ABRB_OK;
}

int abrb_gather_import(abrb_gather *g, int peer_rank, const unsigned char handle[64]) {
  if (!g || !handle) return fail(ABRB_EINVAL, "abrb_gather_import: NULL argument");
  if (peer_rank < 0 || peer_rank >= g->world || peer_rank == g->rank || g->peer[peer_rank])
    return fail(ABRB_EINVAL, "abrb_gather_import: bad or repeated peer rank");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, 64);
  cudaError_t e = cudaIpcOpenMemHandle(&g->peer[peer_rank], h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    g->peer[peer_rank] = nullptr;
    return cuda_fail((int)e, "abrb_gather_import (is peer access between the two GPUs possible?)");
  }
  g->imported[peer_rank] = true;
  return ABRB_OK;
}

void *abrb_gather_buffer(const abrb_gather *g, int buffer_index) {
  if (!g || buffer_index < 0 || buffer_index >= g->n_buffers) return nullptr;
  return static_cast<char *>(g->peer[g->rank]) + (size_t)buffer_index * g->bytes;
}

int abrb_gather_destroy(abrb_gather *g) {
  if (!g) return ABRB_OK;
  int cur = 0;
  cudaGetDevice(&cur);
  cudaSetDevice(g->dev);
  cudaDeviceSynchronize();
  for (int r = 0; r < g->world; ++r)
    if (g->imported[r]) cudaIpcCloseMemHandle(g->peer[r]);
  cudaFree(g->peer[g->rank]);
  cudaSetDevice(cur);
  delete g;
  return ABRB_OK;
}

int abrb_gather_wait(abrb_gather *g, void *stream) {
  if (!g) return fail(ABRB_EINVAL, "abrb_gather_wait: NULL argument");
  char *mine = static_cast<char *>(g->peer[g->rank]);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(1);
  cfg.blockDim = dim3(32);
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gather_wait_kernel,
                                     (const unsigned long long *)reinterpret_cast<unsigned long long *>(mine + g->flag_off),
                                     g->world, g->epoch, reinterpret_cast<int *>(mine + g->counter_off + 64));
  count_launch();
  if (e == cudaSuccess) e = cudaGetLastError();
  return e ? cuda_fail((int)e, "abrb_gather_wait") : ABRB_OK;
}

int abrb_gather_status(const abrb_gather *g) {  // after a stream synchronise: 1 if a wait ever timed out
  if (!g) return fail(ABRB_EINVAL, "abrb_gather_status: NULL argument");
  int st = 0;
  cudaError_t e = cudaMemcpy(&st, static_cast<char *>(g->peer[g->rank]) + g->counter_off + 64, sizeof st, cudaMemcpyDeviceToHost);
  return e ? cuda_fail((int)e, "abrb_gather_status") : st;
}

static int osc_generate_gather(const abrb_osc *c, int frame_id, const double *x_off, const void *q, const void *dq,
                               const void *target, int target_stride, const void *tv, int tv_stride, void *u,
                               void *train, void *ierr, int64_t B, abrb_gather *g, int buffer_index, int64_t row0,
                               void *stream, bool f32) {
  if (!c || !g) return fail(ABRB_EINVAL, "abrb_osc_generate_gather: NULL argument");
  if (buffer_index < 0 || buffer_index >= g->n_buffers || row0 < 0 || B < 0)
    return fail(ABRB_EINVAL, "abrb_osc_generate_gather: bad buffer index / row offset");
  const size_t es = f32 ? 4 : 8, n = (size_t)c->model->host.n;
  if ((size_t)(row0 + B) * n * es > g->bytes)
    return fail(ABRB_EINVAL, "abrb_osc_generate_gather: rows do not fit the gather buffer");
  for (int r = 0; r < g->world; ++r)
    if (!g->peer[r]) return fail(ABRB_EINVAL, "abrb_osc_generate_gather: not every peer has been imported");
  GatherArgs ga;
  ga.n_peer = g->world;
  ga.self = g->rank;
  ga.row0 = row0;
  ga.epoch = ++g->epoch;
  for (int r = 0; r < g->world; ++r) {
    char *base = static_cast<char *>(g->peer[r]);
    ga.peer_u[r] = base + (size_t)buffer_index * g->bytes;
    ga.peer_flag[r] = reinterpret_cast<unsigned long long *>(base + g->flag_off) + g->rank;
  }
  ga.cta_counter = reinterpret_cast<unsigned *>(static_cast<char *>(g->peer[g->rank]) + g->counter_off);
  if (B == 0) {  // an empty shard still has to publish its epoch: the peers wait for it
    for (int r = 0; r < g->world; ++r) {
      cudaError_t e = cudaMemcpyAsync(ga.peer_flag[r], &g->epoch, sizeof(unsigned long long), cudaMemcpyHostToDevice,
                                      (cudaStream_t)stream);
      if (e != cudaSuccess) return cuda_fail((int)e, "abrb_osc_generate_gather(empty shard)");
    }
    return ABRB_OK;
  }
  return osc_generate(c, frame_id, x_off, q, dq, target, target_stride, tv, tv_stride, u, train, ierr, B, stream, f32, &ga);
}

int abrb_osc_generate_gather_f64(const abrb_osc *c, int frame_id, const double *x_off, const double *q, const double *dq,
                                 const double *target, int target_stride, const double *target_velocity, int tv_stride,
                                 double *u, double *training_signal, double *integrated_error, int64_t B,
                                 abrb_gather *g, int buffer_index, int64_t row0, void *stream) {
  return osc_generate_gather(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                             training_signal, integrated_error, B, g, buffer_index, row0, stream, false);
}
int abrb_osc_generate_gather_f32(const abrb_osc *c, int frame_id, const double *x_off, const float *q, const float *dq,
                                 const float *target, int target_stride, const float *target_velocity, int tv_stride,
                                 float *u, float *training_signal, float *integrated_error, int64_t B, abrb_gather *g,
                                 int buffer_index, int64_t row0, void *stream) {
  return osc_generate_gather(c, frame_id, x_off, q, dq, target, target_stride, target_velocity, tv_stride, u,
                             training_signal, integrated_error, B, g, buffer_index, row0, stream, true);
}

// ------------------------------------------------------------------------------------------------ null
static int null_generate(const abrb_model *m, const abrb_null_params *p, const void *q, const void *dq, void *u,
                         int64_t B, void *stream, bool f32) {
  if (!m || !p) return fail(ABRB_EINVAL, "abrb_null_generate: NULL argument");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_null_generate: B < 0");
  std::string e = check_null(m->host.n, *p);
  if (!e.empty()) return fail(ABRB_EUNSUP, "abrb_null_generate: " + e);
  if (B == 0) return ABRB_OK;
  if (!q || !dq || !u) return fail(ABRB_EINVAL, "abrb_null_generate: NULL q/dq/u");
  if (!aligned_elem(q, f32) || !aligned_elem(dq, f32) || !aligned_elem(u, f32))
    return fail(ABRB_EINVAL, "abrb_null_generate: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  NullCall k{q, dq, u, B, f32, (cudaStream_t)stream};
  int ce = cudaErrorInvalidValue;
  switch (m->host.n) {
#define X(j) case j: ce = launch_null<j>(m->host, *p, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return ce ? cuda_fail(ce, "abrb_null_generate") : ABRB_OK;
}

int abrb_null_generate_f64(const abrb_model *m, const abrb_null_params *p, const double *q, const double *dq,
                           double *u, int64_t B, void *stream) {
  return null_generate(m, p, q, dq, u, B, stream, false);
}
int abrb_null_generate_f32(const abrb_model *m, const abrb_null_params *p, const float *q, const float *dq, float *u,
                           int64_t B, void *stream) {
  return null_generate(m, p, q, dq, u, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ sliding
static int sliding_generate(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                            const double *x_off, const void *q, const void *dq, const void *target, int target_stride,
                            const void *tv, int tv_stride, const void *ta, int ta_stride, void *u, void *s, int64_t B,
                            void *stream, bool f32) {
  if (!m) return fail(ABRB_EINVAL, "abrb_sliding_generate: NULL model");
  if (B < 0) return fail(ABRB_EINVAL, "abrb_sliding_generate: B < 0");
  const int n = m->host.n, w = cartesian ? 3 : n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, "abrb_sliding_generate: invalid frame id");
  if ((target_stride != 0 && target_stride != w) || (tv && tv_stride != 0 && tv_stride != w) ||
      (ta && ta_stride != 0 && ta_stride != w))
    return fail(ABRB_EINVAL, "abrb_sliding_generate: stride must be 0 (broadcast) or the row width (3 or n_joints)");
  if (B == 0) return ABRB_OK;
  if (!q || !dq || !target || !u) return fail(ABRB_EINVAL, "abrb_sliding_generate: NULL q/dq/target/u");
  if (!aligned_elem(q, f32) || !aligned_elem(dq, f32) || !aligned_elem(u, f32) || (s && !aligned_elem(s, f32)))
    return fail(ABRB_EINVAL, "abrb_sliding_generate: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  SlidingCall k{kd, lamb, cartesian, frame_id, x_off, q, dq, target, tv, ta, target_stride, tv_stride, ta_stride,
                u, s, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_sliding<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, "abrb_sliding_generate") : ABRB_OK;
}

int abrb_sliding_generate_f64(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                              const double *x_off, const double *q, const double *dq, const double *target,
                              int target_stride, const double *target_velocity, int tv_stride,
                              const double *target_acc, int ta_stride, double *u, double *s, int64_t B, void *stream) {
  return sliding_generate(m, kd, lamb, cartesian, frame_id, x_off, q, dq, target, target_stride, target_velocity,
                          tv_stride, target_acc, ta_stride, u, s, B, stream, false);
}
int abrb_sliding_generate_f32(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                              const double *x_off, const float *q, const float *dq, const float *target,
                              int target_stride, const float *target_velocity, int tv_stride, const float *target_acc,
                              int ta_stride, float *u, float *s, int64_t B, void *stream) {
  return sliding_generate(m, kd, lamb, cartesian, frame_id, x_off, q, dq, target, target_stride, target_velocity,
                          tv_stride, target_acc, ta_stride, u, s, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ inverse kinematics
static int ik_path(const abrb_model *m, double max_dx, double max_dr, double max_dq, int method, double dt, int steps,
                   const void *position, const void *target, int target_stride, void *pos_path, void *vel_path,
                   int64_t B, void *stream, bool f32) {
  if (!m) return fail(ABRB_EINVAL, "abrb_ik_path: NULL model");
  if (B < 0 || steps < 0) return fail(ABRB_EINVAL, "abrb_ik_path: negative size");
  if (method < 1 || method > 3) return fail(ABRB_EUNSUP, "abrb_ik_path: method must be 1, 2 or 3");
  if (target_stride != 0 && target_stride != 6) return fail(ABRB_EINVAL, "abrb_ik_path: stride must be 0 or 6");
  if (B == 0 || steps == 0) return ABRB_OK;
  if (!position || !target || !pos_path || !vel_path) return fail(ABRB_EINVAL, "abrb_ik_path: NULL argument");
  if (!aligned_elem(position, f32) || !aligned_elem(pos_path, f32) || !aligned_elem(vel_path, f32))
    return fail(ABRB_EINVAL, "abrb_ik_path: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  IkCall k{max_dx, max_dr, max_dq, dt, method, steps, position, target, target_stride, pos_path, vel_path, B, f32,
           (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (m->host.n) {
#define X(j) case j: e = launch_ik<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, "abrb_ik_path") : ABRB_OK;
}

int abrb_ik_path_f64(const abrb_model *m, double max_dx, double max_dr, double max_dq, int method, double dt,
                     int n_timesteps, const double *position, const double *target, int target_stride,
                     double *position_path, double *velocity_path, int64_t B, void *stream) {
  return ik_path(m, max_dx, max_dr, max_dq, method, dt, n_timesteps, position, target, target_stride, position_path,
                 velocity_path, B, stream, false);
}
int abrb_ik_path_f32(const abrb_model *m, double max_dx, double max_dr, double max_dq, int method, double dt,
                     int n_timesteps, const float *position, const float *target, int target_stride,
                     float *position_path, float *velocity_path, int64_t B, void *stream) {
  return ik_path(m, max_dx, max_dr, max_dq, method, dt, n_timesteps, position, target, target_stride, position_path,
                 velocity_path, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ joint / floating
static int ctrl_generate(const abrb_model *m, int kind, double kp, double kv, int fa, int fb, const void *q,
                         const void *dq, const void *target, int target_stride, const void *tv, int tv_stride, void *u,
                         int64_t B, void *stream, bool f32, const char *who) {
  if (!m) return fail(ABRB_EINVAL, std::string(who) + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, std::string(who) + ": B < 0");
  const int n = m->host.n;
  if (kind == 0 && ((target_stride != 0 && target_stride != n) || (tv && tv_stride != 0 && tv_stride != n)))
    return fail(ABRB_EINVAL, std::string(who) + ": stride must be 0 (broadcast) or n_joints");
  if (B == 0) return ABRB_OK;
  if (!q || !u || (kind == 0 && (!dq || !target)) || (kind == 1 && fb && !dq))
    return fail(ABRB_EINVAL, std::string(who) + ": NULL q/dq/target/u");
  if (!aligned_elem(q, f32) || !aligned_elem(u, f32) || (dq && !aligned_elem(dq, f32)))
    return fail(ABRB_EINVAL, std::string(who) + ": misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  CtrlCall k{kind, kp, kv, fa, fb, q, dq, target, tv, target_stride, tv_stride, u, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_ctrl<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_joint_generate_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, const double *q,
                            const double *dq, const double *target, int target_stride, const double *target_velocity,
                            int tv_stride, double *u, int64_t B, void *stream) {
  return ctrl_generate(m, 0, kp, kv, account_for_gravity, 0, q, dq, target, target_stride, target_velocity, tv_stride, u,
                       B, stream, false, "abrb_joint_generate");
}
int abrb_joint_generate_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, const float *q,
                            const float *dq, const float *target, int target_stride, const float *target_velocity,
                            int tv_stride, float *u, int64_t B, void *stream) {
  return ctrl_generate(m, 0, kp, kv, account_for_gravity, 0, q, dq, target, target_stride, target_velocity, tv_stride, u,
                       B, stream, true, "abrb_joint_generate");
}
int abrb_floating_generate_f64(const abrb_model *m, int task_space, int dynamic, const double *q, const double *dq,
                               double *u, int64_t B, void *stream) {
  return ctrl_generate(m, 1, 0, 0, task_space, dynamic, q, dq, nullptr, 0, nullptr, 0, u, B, stream, false,
                       "abrb_floating_generate");
}
int abrb_floating_generate_f32(const abrb_model *m, int task_space, int dynamic, const float *q, const float *dq, float *u,
                               int64_t B, void *stream) {
  return ctrl_generate(m, 1, 0, 0, task_space, dynamic, q, dq, nullptr, 0, nullptr, 0, u, B, stream, true,
                       "abrb_floating_generate");
}

// ------------------------------------------------------------------------------------------------ rollout
static int osc_rollout(const abrb_osc *c, int frame_id, const double *x_off, void *q, void *dq, const void *target,
                       int target_stride, int steps, double dt, void *q_traj, void *dq_traj, void *u_traj, void *ierr,
                       int64_t B, void *stream, bool f32) {
  if (!c) return fail(ABRB_EINVAL, "abrb_osc_rollout: NULL controller");
  if (B < 0 || steps < 0) return fail(ABRB_EINVAL, "abrb_osc_rollout: B < 0 or steps < 0");
  const int n = c->model->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, "abrb_osc_rollout: invalid frame id");
  if (target_stride != 0 && target_stride != 6) return fail(ABRB_EINVAL, "abrb_osc_rollout: stride must be 0 or 6");
  if ((c->params.ki != 0.0) != (ierr != nullptr))
    return fail(ABRB_EINVAL, "abrb_osc_rollout: integrated_error must be given if and only if ki != 0");
  if (B == 0 || steps == 0) return ABRB_OK;
  if (!q || !dq || !target) return fail(ABRB_EINVAL, "abrb_osc_rollout: NULL q/dq/target");
  const void *ptrs[] = {q, dq, target, q_traj, dq_traj, u_traj, ierr};
  for (const void *p : ptrs)
    if (p && !aligned_elem(p, f32)) return fail(ABRB_EINVAL, "abrb_osc_rollout: misaligned pointer");
  int rc = ensure_device();
  if (rc) return rc;
  RolloutCall k{frame_id, x_off, q, dq, target, target_stride, steps, dt, q_traj, dq_traj, u_traj, B, f32, (cudaStream_t)stream};
  k.ierr = ierr;
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_rollout<j>(c->model->host, c->params, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, "abrb_osc_rollout") : ABRB_OK;
}

int abrb_osc_rollout_f64(const abrb_osc *c, int frame_id, const double *x_off, double *q, double *dq,
                         const double *target, int target_stride, int steps, double dt, double *q_traj,
                         double *dq_traj, double *u_traj, double *integrated_error, int64_t B, void *stream) {
  return osc_rollout(c, frame_id, x_off, q, dq, target, target_stride, steps, dt, q_traj, dq_traj, u_traj,
                     integrated_error, B, stream, false);
}
int abrb_osc_rollout_f32(const abrb_osc *c, int frame_id, const double *x_off, float *q, float *dq, const float *target,
                         int target_stride, int steps, double dt, float *q_traj, float *dq_traj, float *u_traj,
                         float *integrated_error, int64_t B, void *stream) {
  return osc_rollout(c, frame_id, x_off, q, dq, target, target_stride, steps, dt, q_traj, dq_traj, u_traj,
                     integrated_error, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ path rollout
static int osc_rollout_path(const abrb_osc *c, int frame_id, const double *x_off, void *q, void *dq, const void *path,
                            int path_stride, const void *path_velocity, int pv_stride, int steps, double dt,
                            double effort_weight, void *q_traj, void *dq_traj, void *u_traj, void *x_traj, void *cost,
                            void *ierr, int64_t B, void *stream, bool f32) {
  const char *who = "abrb_osc_rollout_path";
  const std::string w(who);
  if (!c) return fail(ABRB_EINVAL, w + ": NULL controller");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = c->model->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, w + ": invalid frame id");
  if (path_stride != 0 && path_stride != 6) return fail(ABRB_EINVAL, w + ": path_stride must be 0 or 6");
  if (pv_stride != 0 && pv_stride != 6) return fail(ABRB_EINVAL, w + ": pv_stride must be 0 or 6");
  if (!std::isfinite(effort_weight) || effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if ((c->params.ki != 0.0) != (ierr != nullptr))
    return fail(ABRB_EINVAL, w + ": integrated_error must be given if and only if ki != 0");
  if (B == 0) return ABRB_OK;
  if (!q) return fail(ABRB_EINVAL, w + ": NULL q");
  if (!dq) return fail(ABRB_EINVAL, w + ": NULL dq");
  if (steps > 0 && !path) return fail(ABRB_EINVAL, w + ": NULL path");
  const void *ptrs[] = {q, dq, path, path_velocity, q_traj, dq_traj, u_traj, x_traj, cost, ierr};
  const char *names[] = {"q", "dq", "path", "path_velocity", "q_traj", "dq_traj", "u_traj", "x_traj", "cost",
                         "integrated_error"};
  for (int i = 0; i < 10; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  if (steps == 0) {  // nothing to step: q, dq and the integrator stay as they are, the cost is zero
    int e = cost ? (int)cudaMemsetAsync(cost, 0, (size_t)B * (f32 ? 4 : 8), (cudaStream_t)stream) : 0;
    return e ? cuda_fail(e, who) : ABRB_OK;
  }
  RolloutPathCall k;
  k.frame = frame_id;
  k.xoff = x_off;
  k.q = q;
  k.dq = dq;
  k.target = path;
  k.target_stride = path_stride;
  k.steps = steps;
  k.dt = dt;
  k.q_traj = q_traj;
  k.dq_traj = dq_traj;
  k.u_traj = u_traj;
  k.B = B;
  k.f32 = f32;
  k.stream = (cudaStream_t)stream;
  k.ierr = ierr;
  k.tv = path_velocity;
  k.tv_stride = pv_stride;
  k.x_traj = x_traj;
  k.cost = cost;
  k.effort_weight = effort_weight;
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_rollout_path<j>(c->model->host, c->params, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_osc_rollout_path_f64(const abrb_osc *c, int frame_id, const double *x_off, double *q, double *dq,
                              const double *path, int path_stride, const double *path_velocity, int pv_stride,
                              int steps, double dt, double effort_weight, double *q_traj, double *dq_traj,
                              double *u_traj, double *x_traj, double *cost, double *integrated_error, int64_t B,
                              void *stream) {
  return osc_rollout_path(c, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride, steps, dt,
                          effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, integrated_error, B, stream, false);
}
int abrb_osc_rollout_path_f32(const abrb_osc *c, int frame_id, const double *x_off, float *q, float *dq,
                              const float *path, int path_stride, const float *path_velocity, int pv_stride,
                              int steps, double dt, double effort_weight, float *q_traj, float *dq_traj,
                              float *u_traj, float *x_traj, float *cost, float *integrated_error, int64_t B,
                              void *stream) {
  return osc_rollout_path(c, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride, steps, dt,
                          effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, integrated_error, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ plant
static int plant_dynamics(const abrb_model *m, const void *q, const void *dq, const void *in, void *out, int64_t B,
                          void *stream, bool f32, int kind) {
  const char *who = kind == 0 ? "abrb_forward_dynamics" : "abrb_inverse_dynamics";
  const char *in_name = kind == 0 ? "u" : "ddq", *out_name = kind == 0 ? "ddq" : "u";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (B == 0) return ABRB_OK;
  const void *ptrs[] = {q, dq, in, out};
  const char *names[] = {"q", "dq", in_name, out_name};
  for (int i = 0; i < 4; ++i) {
    if (!ptrs[i]) return fail(ABRB_EINVAL, w + ": NULL " + names[i]);
    if (!aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  }
  int rc = ensure_device();
  if (rc) return rc;
  DynCall k{kind, q, dq, in, out, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (m->host.n) {
#define X(j) case j: e = launch_dyn<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_forward_dynamics_f64(const abrb_model *m, const double *q, const double *dq, const double *u, double *ddq,
                              int64_t B, void *stream) {
  return plant_dynamics(m, q, dq, u, ddq, B, stream, false, 0);
}
int abrb_forward_dynamics_f32(const abrb_model *m, const float *q, const float *dq, const float *u, float *ddq,
                              int64_t B, void *stream) {
  return plant_dynamics(m, q, dq, u, ddq, B, stream, true, 0);
}
int abrb_inverse_dynamics_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq, double *u,
                              int64_t B, void *stream) {
  return plant_dynamics(m, q, dq, ddq, u, B, stream, false, 1);
}
int abrb_inverse_dynamics_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq, float *u,
                              int64_t B, void *stream) {
  return plant_dynamics(m, q, dq, ddq, u, B, stream, true, 1);
}

static int dynamics_regressor(const abrb_model *m, const void *q, const void *dq, const void *ddq, void *Yt, int64_t B,
                              void *stream, bool f32) {
  const char *who = "abrb_inverse_dynamics_regressor";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (B == 0) return ABRB_OK;
  const void *ptrs[] = {q, dq, ddq, Yt};
  const char *names[] = {"q", "dq", "ddq", "Yt"};
  for (int i = 0; i < 4; ++i) {
    if (!ptrs[i]) return fail(ABRB_EINVAL, w + ": NULL " + names[i]);
    if (!aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  }
  int rc = ensure_device();
  if (rc) return rc;
  RegressorCall k{q, dq, ddq, Yt, B, m->desc.gravity, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (m->host.n) {
#define X(j) case j: e = launch_regressor<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_inverse_dynamics_regressor_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq,
                                        double *Yt, int64_t B, void *stream) {
  return dynamics_regressor(m, q, dq, ddq, Yt, B, stream, false);
}
int abrb_inverse_dynamics_regressor_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq,
                                        float *Yt, int64_t B, void *stream) {
  return dynamics_regressor(m, q, dq, ddq, Yt, B, stream, true);
}

static int plant_rollout(const abrb_model *m, int frame_id, const double *x_off, void *q, void *dq, const void *u,
                         int u_stride, int compensate_gravity, const void *path, int path_stride, int steps, double dt,
                         double effort_weight, void *q_traj, void *dq_traj, void *u_traj, void *x_traj, void *cost,
                         int64_t B, void *stream, bool f32) {
  const char *who = "abrb_plant_rollout";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = m->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, w + ": invalid frame id");
  if (u_stride != 0 && u_stride != n) return fail(ABRB_EINVAL, w + ": u_stride must be 0 or n_joints");
  if (path_stride != 0 && path_stride != 6) return fail(ABRB_EINVAL, w + ": path_stride must be 0 or 6");
  if (!std::isfinite(effort_weight) || effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if (B == 0) return ABRB_OK;
  if (!q) return fail(ABRB_EINVAL, w + ": NULL q");
  if (!dq) return fail(ABRB_EINVAL, w + ": NULL dq");
  if (steps > 0 && !u) return fail(ABRB_EINVAL, w + ": NULL u");
  const void *ptrs[] = {q, dq, u, path, q_traj, dq_traj, u_traj, x_traj, cost};
  const char *names[] = {"q", "dq", "u", "path", "q_traj", "dq_traj", "u_traj", "x_traj", "cost"};
  for (int i = 0; i < 9; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  if (steps == 0) {  // nothing to step: q and dq stay as they are, the cost is zero
    int e = cost ? (int)cudaMemsetAsync(cost, 0, (size_t)B * (f32 ? 4 : 8), (cudaStream_t)stream) : 0;
    return e ? cuda_fail(e, who) : ABRB_OK;
  }
  PlantCall k{frame_id, x_off, q, dq, u, u_stride, compensate_gravity, path, path_stride, steps, dt, effort_weight,
              q_traj, dq_traj, u_traj, x_traj, cost, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_plant<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_plant_rollout_f64(const abrb_model *m, int frame_id, const double *x_off, double *q, double *dq,
                           const double *u, int u_stride, int compensate_gravity, const double *path, int path_stride,
                           int steps, double dt, double effort_weight, double *q_traj, double *dq_traj, double *u_traj,
                           double *x_traj, double *cost, int64_t B, void *stream) {
  return plant_rollout(m, frame_id, x_off, q, dq, u, u_stride, compensate_gravity, path, path_stride, steps, dt,
                       effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream, false);
}
int abrb_plant_rollout_f32(const abrb_model *m, int frame_id, const double *x_off, float *q, float *dq, const float *u,
                           int u_stride, int compensate_gravity, const float *path, int path_stride, int steps,
                           double dt, double effort_weight, float *q_traj, float *dq_traj, float *u_traj,
                           float *x_traj, float *cost, int64_t B, void *stream) {
  return plant_rollout(m, frame_id, x_off, q, dq, u, u_stride, compensate_gravity, path, path_stride, steps, dt,
                       effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream, true);
}

// ------------------------------------------------------------------------------------------------ Joint / Sliding rollouts
// `k` carries the controller (kind, gains, flags), the frame and the records; its path strides are checked here against
// the row width w (3 for cartesian Sliding, n_joints otherwise)
static int ctrl_rollout(const abrb_model *m, CtrlRolloutCall k, const char *who) {
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (k.B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (k.steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = m->host.n;
  if (k.frame < 0 || k.frame > 2 * n + 1) return fail(ABRB_EFRAME, w + ": invalid frame id");
  const bool task = k.kind == kCtrlSliding && k.cartesian;
  const int width = task ? 3 : n;
  const char *wname = task ? "3 (cartesian)" : "n_joints";
  const int strides[] = {k.path_stride, k.pv_stride, k.pa_stride};
  const char *snames[] = {"path_stride", "pv_stride", "pa_stride"};
  for (int i = 0; i < (k.kind == kCtrlSliding ? 3 : 2); ++i)
    if (strides[i] != 0 && strides[i] != width) return fail(ABRB_EINVAL, w + ": " + snames[i] + " must be 0 or " + wname);
  if (!std::isfinite(k.effort_weight) || k.effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if (k.B == 0) return ABRB_OK;
  if (!k.q) return fail(ABRB_EINVAL, w + ": NULL q");
  if (!k.dq) return fail(ABRB_EINVAL, w + ": NULL dq");
  if (k.steps > 0 && !k.path) return fail(ABRB_EINVAL, w + ": NULL path");
  const void *ptrs[] = {k.q, k.dq, k.path, k.pv, k.pa, k.q_traj, k.dq_traj, k.u_traj, k.x_traj, k.cost};
  const char *names[] = {"q", "dq", "path", "path_velocity", "path_acc", "q_traj", "dq_traj", "u_traj", "x_traj",
                         "cost"};
  for (int i = 0; i < 10; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], k.f32))
      return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  if (k.steps == 0) {  // nothing to step: q and dq stay as they are, the cost is zero
    int e = k.cost ? (int)cudaMemsetAsync(k.cost, 0, (size_t)k.B * (k.f32 ? 4 : 8), k.stream) : 0;
    return e ? cuda_fail(e, who) : ABRB_OK;
  }
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_ctrl_rollout<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

static int joint_rollout(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                         const double *x_off, void *q, void *dq, const void *path, int path_stride,
                         const void *path_velocity, int pv_stride, int steps, double dt, double effort_weight,
                         void *q_traj, void *dq_traj, void *u_traj, void *x_traj, void *cost, int64_t B, void *stream,
                         bool f32) {
  CtrlRolloutCall k{kCtrlJoint, kp, kv, account_for_gravity, 0.0, 0.0, 0, frame_id, x_off, q, dq, path,
                    path_velocity, nullptr, path_stride, pv_stride, 0, steps, dt, effort_weight, q_traj, dq_traj,
                    u_traj, x_traj, cost, B, f32, (cudaStream_t)stream};
  return ctrl_rollout(m, k, "abrb_joint_rollout_path");
}

static int sliding_rollout(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                           const double *x_off, void *q, void *dq, const void *path, int path_stride,
                           const void *path_velocity, int pv_stride, const void *path_acc, int pa_stride, int steps,
                           double dt, double effort_weight, void *q_traj, void *dq_traj, void *u_traj, void *x_traj,
                           void *cost, int64_t B, void *stream, bool f32) {
  CtrlRolloutCall k{kCtrlSliding, 0.0, 0.0, 0, kd, lamb, cartesian != 0, frame_id, x_off, q, dq, path, path_velocity,
                    path_acc, path_stride, pv_stride, pa_stride, steps, dt, effort_weight, q_traj, dq_traj, u_traj,
                    x_traj, cost, B, f32, (cudaStream_t)stream};
  return ctrl_rollout(m, k, "abrb_sliding_rollout_path");
}

int abrb_joint_rollout_path_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                const double *x_off, double *q, double *dq, const double *path, int path_stride,
                                const double *path_velocity, int pv_stride, int steps, double dt,
                                double effort_weight, double *q_traj, double *dq_traj, double *u_traj,
                                double *x_traj, double *cost, int64_t B, void *stream) {
  return joint_rollout(m, kp, kv, account_for_gravity, frame_id, x_off, q, dq, path, path_stride, path_velocity,
                       pv_stride, steps, dt, effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream, false);
}
int abrb_joint_rollout_path_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                const double *x_off, float *q, float *dq, const float *path, int path_stride,
                                const float *path_velocity, int pv_stride, int steps, double dt, double effort_weight,
                                float *q_traj, float *dq_traj, float *u_traj, float *x_traj, float *cost, int64_t B,
                                void *stream) {
  return joint_rollout(m, kp, kv, account_for_gravity, frame_id, x_off, q, dq, path, path_stride, path_velocity,
                       pv_stride, steps, dt, effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream, true);
}
int abrb_sliding_rollout_path_f64(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                                  const double *x_off, double *q, double *dq, const double *path, int path_stride,
                                  const double *path_velocity, int pv_stride, const double *path_acc, int pa_stride,
                                  int steps, double dt, double effort_weight, double *q_traj, double *dq_traj,
                                  double *u_traj, double *x_traj, double *cost, int64_t B, void *stream) {
  return sliding_rollout(m, kd, lamb, cartesian, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride,
                         path_acc, pa_stride, steps, dt, effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B,
                         stream, false);
}
int abrb_sliding_rollout_path_f32(const abrb_model *m, double kd, double lamb, int cartesian, int frame_id,
                                  const double *x_off, float *q, float *dq, const float *path, int path_stride,
                                  const float *path_velocity, int pv_stride, const float *path_acc, int pa_stride,
                                  int steps, double dt, double effort_weight, float *q_traj, float *dq_traj,
                                  float *u_traj, float *x_traj, float *cost, int64_t B, void *stream) {
  return sliding_rollout(m, kd, lamb, cartesian, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride,
                         path_acc, pa_stride, steps, dt, effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B,
                         stream, true);
}


// ------------------------------------------------------------------------------------------------ plant derivatives
static int dynamics_derivatives(const abrb_model *m, const void *q, const void *dq, const void *in, void *d_q,
                                void *d_dq, void *d_in, int64_t B, void *stream, bool f32, int kind) {
  const char *who = kind == 0 ? "abrb_forward_dynamics_derivatives" : "abrb_inverse_dynamics_derivatives";
  const char *in_name = kind == 0 ? "u" : "ddq", *d_in_name = kind == 0 ? "d_u" : "d_ddq";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (B == 0) return ABRB_OK;
  const void *ptrs[] = {q, dq, in, d_q, d_dq};
  const char *names[] = {"q", "dq", in_name, "d_q", "d_dq"};
  for (int i = 0; i < 5; ++i) {
    if (!ptrs[i]) return fail(ABRB_EINVAL, w + ": NULL " + names[i]);
    if (!aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  }
  if (d_in && !aligned_elem(d_in, f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + d_in_name + ")");
  int rc = ensure_device();
  if (rc) return rc;
  DynJacCall k{kind, q, dq, in, d_q, d_dq, d_in, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (m->host.n) {
#define X(j) case j: e = launch_dyn_jac<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_forward_dynamics_derivatives_f64(const abrb_model *m, const double *q, const double *dq, const double *u,
                                          double *d_q, double *d_dq, double *d_u, int64_t B, void *stream) {
  return dynamics_derivatives(m, q, dq, u, d_q, d_dq, d_u, B, stream, false, 0);
}
int abrb_forward_dynamics_derivatives_f32(const abrb_model *m, const float *q, const float *dq, const float *u,
                                          float *d_q, float *d_dq, float *d_u, int64_t B, void *stream) {
  return dynamics_derivatives(m, q, dq, u, d_q, d_dq, d_u, B, stream, true, 0);
}
int abrb_inverse_dynamics_derivatives_f64(const abrb_model *m, const double *q, const double *dq, const double *ddq,
                                          double *d_q, double *d_dq, double *d_ddq, int64_t B, void *stream) {
  return dynamics_derivatives(m, q, dq, ddq, d_q, d_dq, d_ddq, B, stream, false, 1);
}
int abrb_inverse_dynamics_derivatives_f32(const abrb_model *m, const float *q, const float *dq, const float *ddq,
                                          float *d_q, float *d_dq, float *d_ddq, int64_t B, void *stream) {
  return dynamics_derivatives(m, q, dq, ddq, d_q, d_dq, d_ddq, B, stream, true, 1);
}

static int plant_rollout_vjp(const abrb_model *m, int frame_id, const double *x_off, const void *q0, const void *dq0,
                             const void *u, int u_stride, int compensate_gravity, const void *path, int path_stride,
                             int steps, double dt, double effort_weight, const void *q_traj, const void *dq_traj,
                             const void *g_cost, const void *g_q, const void *g_dq, const void *g_q_traj,
                             const void *g_dq_traj, const void *g_u_traj, const void *g_x_traj, void *gu, void *gq0,
                             void *gdq0, int64_t B, void *stream, bool f32) {
  const char *who = "abrb_plant_rollout_vjp";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = m->host.n;
  if (frame_id < 0 || frame_id > 2 * n + 1) return fail(ABRB_EFRAME, w + ": invalid frame id");
  if (u_stride != 0 && u_stride != n) return fail(ABRB_EINVAL, w + ": u_stride must be 0 or n_joints");
  if (path_stride != 0 && path_stride != 6) return fail(ABRB_EINVAL, w + ": path_stride must be 0 or 6");
  if (!std::isfinite(effort_weight) || effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if (B == 0) return ABRB_OK;
  if (!q0) return fail(ABRB_EINVAL, w + ": NULL q0");
  if (!dq0) return fail(ABRB_EINVAL, w + ": NULL dq0");
  if (!gq0) return fail(ABRB_EINVAL, w + ": NULL gq0");
  if (!gdq0) return fail(ABRB_EINVAL, w + ": NULL gdq0");
  if (steps > 0) {
    if (!u) return fail(ABRB_EINVAL, w + ": NULL u");
    if (!q_traj) return fail(ABRB_EINVAL, w + ": NULL q_traj");
    if (!dq_traj) return fail(ABRB_EINVAL, w + ": NULL dq_traj");
    if (!gu) return fail(ABRB_EINVAL, w + ": NULL gu");
  }
  const void *ptrs[] = {q0, dq0, u, path, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj,
                        gu, gq0, gdq0};
  const char *names[] = {"q0", "dq0", "u", "path", "q_traj", "dq_traj", "g_cost", "g_q", "g_dq", "g_q_traj",
                         "g_dq_traj", "g_u_traj", "g_x_traj", "gu", "gq0", "gdq0"};
  for (int i = 0; i < 16; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  PlantVjpCall k{frame_id, x_off, q0, dq0, u, u_stride, compensate_gravity, path, path_stride, steps, dt,
                 effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj,
                 gu, gq0, gdq0, B, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_plant_vjp<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_plant_rollout_vjp_f64(const abrb_model *m, int frame_id, const double *x_off, const double *q0,
                               const double *dq0, const double *u, int u_stride, int compensate_gravity,
                               const double *path, int path_stride, int steps, double dt, double effort_weight,
                               const double *q_traj, const double *dq_traj, const double *g_cost, const double *g_q,
                               const double *g_dq, const double *g_q_traj, const double *g_dq_traj,
                               const double *g_u_traj, const double *g_x_traj, double *gu, double *gq0, double *gdq0,
                               int64_t B, void *stream) {
  return plant_rollout_vjp(m, frame_id, x_off, q0, dq0, u, u_stride, compensate_gravity, path, path_stride, steps, dt,
                           effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj,
                           gu, gq0, gdq0, B, stream, false);
}
int abrb_plant_rollout_vjp_f32(const abrb_model *m, int frame_id, const double *x_off, const float *q0,
                               const float *dq0, const float *u, int u_stride, int compensate_gravity,
                               const float *path, int path_stride, int steps, double dt, double effort_weight,
                               const float *q_traj, const float *dq_traj, const float *g_cost, const float *g_q,
                               const float *g_dq, const float *g_q_traj, const float *g_dq_traj,
                               const float *g_u_traj, const float *g_x_traj, float *gu, float *gq0, float *gdq0,
                               int64_t B, void *stream) {
  return plant_rollout_vjp(m, frame_id, x_off, q0, dq0, u, u_stride, compensate_gravity, path, path_stride, steps, dt,
                           effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj,
                           gu, gq0, gdq0, B, stream, true);
}

static int plant_rollout_theta_vjp(const abrb_model *m, const void *q0, const void *dq0, const void *u, int u_stride,
                                   int compensate_gravity, int steps, double effort_weight, const void *q_traj,
                                   const void *dq_traj, const void *gu, const void *g_cost, const void *g_u_traj,
                                   void *g_theta, int64_t B, void *stream, bool f32) {
  const char *who = "abrb_plant_rollout_theta_vjp";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = m->host.n;
  if (u_stride != 0 && u_stride != n) return fail(ABRB_EINVAL, w + ": u_stride must be 0 or n_joints");
  if (!std::isfinite(effort_weight) || effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if (B == 0) return ABRB_OK;
  if (!q0) return fail(ABRB_EINVAL, w + ": NULL q0");
  if (!dq0) return fail(ABRB_EINVAL, w + ": NULL dq0");
  if (!g_theta) return fail(ABRB_EINVAL, w + ": NULL g_theta");
  if (steps > 0) {
    if (!u) return fail(ABRB_EINVAL, w + ": NULL u");
    if (!q_traj) return fail(ABRB_EINVAL, w + ": NULL q_traj");
    if (!dq_traj) return fail(ABRB_EINVAL, w + ": NULL dq_traj");
    if (!gu) return fail(ABRB_EINVAL, w + ": NULL gu");
  }
  const void *ptrs[] = {q0, dq0, u, q_traj, dq_traj, gu, g_cost, g_u_traj, g_theta};
  const char *names[] = {"q0", "dq0", "u", "q_traj", "dq_traj", "gu", "g_cost", "g_u_traj", "g_theta"};
  for (int i = 0; i < 9; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], f32)) return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  ThetaVjpCall k{q0, dq0, u, u_stride, compensate_gravity, steps, effort_weight, q_traj, dq_traj, gu, g_cost, g_u_traj,
                 g_theta, B, m->desc.gravity, f32, (cudaStream_t)stream};
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_theta_vjp<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_plant_rollout_theta_vjp_f64(const abrb_model *m, const double *q0, const double *dq0, const double *u,
                                     int u_stride, int compensate_gravity, int steps, double effort_weight,
                                     const double *q_traj, const double *dq_traj, const double *gu,
                                     const double *g_cost, const double *g_u_traj, double *g_theta, int64_t B,
                                     void *stream) {
  return plant_rollout_theta_vjp(m, q0, dq0, u, u_stride, compensate_gravity, steps, effort_weight, q_traj, dq_traj,
                                 gu, g_cost, g_u_traj, g_theta, B, stream, false);
}
int abrb_plant_rollout_theta_vjp_f32(const abrb_model *m, const float *q0, const float *dq0, const float *u,
                                     int u_stride, int compensate_gravity, int steps, double effort_weight,
                                     const float *q_traj, const float *dq_traj, const float *gu, const float *g_cost,
                                     const float *g_u_traj, float *g_theta, int64_t B, void *stream) {
  return plant_rollout_theta_vjp(m, q0, dq0, u, u_stride, compensate_gravity, steps, effort_weight, q_traj, dq_traj,
                                 gu, g_cost, g_u_traj, g_theta, B, stream, true);
}

static int joint_rollout_vjp(const abrb_model *m, JointVjpCall k) {
  const char *who = "abrb_joint_rollout_path_vjp";
  const std::string w(who);
  if (!m) return fail(ABRB_EINVAL, w + ": NULL model");
  if (k.B < 0) return fail(ABRB_EINVAL, w + ": B < 0");
  if (k.steps < 0) return fail(ABRB_EINVAL, w + ": steps < 0");
  const int n = m->host.n;
  if (k.frame < 0 || k.frame > 2 * n + 1) return fail(ABRB_EFRAME, w + ": invalid frame id");
  if (k.path_stride != 0 && k.path_stride != n) return fail(ABRB_EINVAL, w + ": path_stride must be 0 or n_joints");
  if (k.pv_stride != 0 && k.pv_stride != n) return fail(ABRB_EINVAL, w + ": pv_stride must be 0 or n_joints");
  if (!std::isfinite(k.effort_weight) || k.effort_weight < 0.0)
    return fail(ABRB_EINVAL, w + ": effort_weight must be finite and >= 0");
  if (k.B == 0) return ABRB_OK;
  if (!k.q0) return fail(ABRB_EINVAL, w + ": NULL q0");
  if (!k.dq0) return fail(ABRB_EINVAL, w + ": NULL dq0");
  if (!k.gq0) return fail(ABRB_EINVAL, w + ": NULL gq0");
  if (!k.gdq0) return fail(ABRB_EINVAL, w + ": NULL gdq0");
  if (k.steps > 0) {
    if (!k.path) return fail(ABRB_EINVAL, w + ": NULL path");
    if (!k.q_traj) return fail(ABRB_EINVAL, w + ": NULL q_traj");
    if (!k.dq_traj) return fail(ABRB_EINVAL, w + ": NULL dq_traj");
  }
  if (k.g_pv && !k.pv) return fail(ABRB_EINVAL, w + ": g_path_velocity without path_velocity");
  const void *ptrs[] = {k.q0, k.dq0, k.path, k.pv, k.q_traj, k.dq_traj, k.g_cost, k.g_q, k.g_dq, k.g_q_traj,
                        k.g_dq_traj, k.g_u_traj, k.g_x_traj, k.g_path, k.g_pv, k.g_gains, k.gq0, k.gdq0};
  const char *names[] = {"q0", "dq0", "path", "path_velocity", "q_traj", "dq_traj", "g_cost", "g_q", "g_dq",
                         "g_q_traj", "g_dq_traj", "g_u_traj", "g_x_traj", "g_path", "g_path_velocity", "g_gains",
                         "gq0", "gdq0"};
  for (int i = 0; i < 18; ++i)
    if (ptrs[i] && !aligned_elem(ptrs[i], k.f32))
      return fail(ABRB_EINVAL, w + ": misaligned pointer (" + names[i] + ")");
  int rc = ensure_device();
  if (rc) return rc;
  int e = cudaErrorInvalidValue;
  switch (n) {
#define X(j) case j: e = launch_joint_vjp<j>(m->host, k); break;
    ABRB_EACH_N(X)
#undef X
  }
  return e ? cuda_fail(e, who) : ABRB_OK;
}

int abrb_joint_rollout_path_vjp_f64(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                    const double *x_off, const double *q0, const double *dq0, const double *path,
                                    int path_stride, const double *path_velocity, int pv_stride, int steps, double dt,
                                    double effort_weight, const double *q_traj, const double *dq_traj,
                                    const double *g_cost, const double *g_q, const double *g_dq,
                                    const double *g_q_traj, const double *g_dq_traj, const double *g_u_traj,
                                    const double *g_x_traj, double *g_path, double *g_path_velocity, double *g_gains,
                                    double *gq0, double *gdq0, int64_t B, void *stream) {
  return joint_rollout_vjp(m, {kp, kv, account_for_gravity, frame_id, x_off, q0, dq0, path, path_velocity, path_stride,
                               pv_stride, steps, dt, effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj,
                               g_dq_traj, g_u_traj, g_x_traj, g_path, g_path_velocity, g_gains, gq0, gdq0, B, false,
                               (cudaStream_t)stream});
}
int abrb_joint_rollout_path_vjp_f32(const abrb_model *m, double kp, double kv, int account_for_gravity, int frame_id,
                                    const double *x_off, const float *q0, const float *dq0, const float *path,
                                    int path_stride, const float *path_velocity, int pv_stride, int steps, double dt,
                                    double effort_weight, const float *q_traj, const float *dq_traj,
                                    const float *g_cost, const float *g_q, const float *g_dq, const float *g_q_traj,
                                    const float *g_dq_traj, const float *g_u_traj, const float *g_x_traj,
                                    float *g_path, float *g_path_velocity, float *g_gains, float *gq0, float *gdq0,
                                    int64_t B, void *stream) {
  return joint_rollout_vjp(m, {kp, kv, account_for_gravity, frame_id, x_off, q0, dq0, path, path_velocity, path_stride,
                               pv_stride, steps, dt, effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj,
                               g_dq_traj, g_u_traj, g_x_traj, g_path, g_path_velocity, g_gains, gq0, gdq0, B, true,
                               (cudaStream_t)stream});
}

// ------------------------------------------------------------------------------------------------ path planner
static int path_check(const char *w, const abrb_path_params *p, const double *table, const double *start,
                      const double *target, const void *a, const void *b, int64_t B) {
  if (!p) return fail(ABRB_EINVAL, std::string(w) + ": NULL params");
  if (B < 0) return fail(ABRB_EINVAL, std::string(w) + ": negative size");
  if (p->vel_kind != ABRB_VEL_GAUSSIAN && p->vel_kind != ABRB_VEL_LINEAR)
    return fail(ABRB_EUNSUP, std::string(w) + ": unknown velocity profile kind");
  if (p->n_points < 2) return fail(ABRB_EINVAL, std::string(w) + ": n_points must be at least 2");
  if (p->n_points > ABRB_PATH_MAX_POINTS)
    return fail(ABRB_EUNSUP, std::string(w) + ": n_points above " + std::to_string(ABRB_PATH_MAX_POINTS) +
                                 " (phase 2 keeps the warped curve in shared memory)");
  if (p->axes[0] < 0 || p->axes[0] > 2)
    return fail(ABRB_EUNSUP, std::string(w) + ": unknown Euler axes (first axis)");
  for (int i = 1; i < 4; ++i)
    if (p->axes[i] != 0 && p->axes[i] != 1) return fail(ABRB_EUNSUP, std::string(w) + ": unknown Euler axes");
  if (!(p->dt > 0.0) || !(p->acceleration > 0.0) || !std::isfinite(p->dt) || !std::isfinite(p->acceleration) ||
      (p->vel_kind == ABRB_VEL_GAUSSIAN && (!(p->n_sigma > 0.0) || !std::isfinite(p->n_sigma))))
    return fail(ABRB_EINVAL, std::string(w) + ": dt, acceleration and n_sigma must be positive and finite");
  if (B == 0) return ABRB_OK;
  const void *ptrs[] = {table, start, target, a, b};
  for (const void *q : ptrs) {
    if (!q) return fail(ABRB_EINVAL, std::string(w) + ": NULL argument");
    if (!aligned_elem(q, false)) return fail(ABRB_EINVAL, std::string(w) + ": misaligned pointer");
  }
  return ABRB_OK;
}

int abrb_path_plan(const abrb_path_params *p, const double *table, const double *start, const double *target,
                   const double *max_velocity, const double *start_velocity, const double *target_velocity,
                   int64_t *lengths, abrb_path_rec *plan, int64_t B, void *stream) {
  const char *w = "abrb_path_plan";
  int rc = path_check(w, p, table, start, target, start_velocity, target_velocity, B);
  if (rc || B == 0) return rc;
  const void *ptrs[] = {max_velocity, lengths, plan};
  for (const void *q : ptrs) {
    if (!q) return fail(ABRB_EINVAL, std::string(w) + ": NULL argument");
    if (!aligned_elem(q, false)) return fail(ABRB_EINVAL, std::string(w) + ": misaligned pointer");
  }
  if ((rc = ensure_device())) return rc;
  PathCall c{*p, table, start, target, max_velocity, start_velocity, target_velocity, nullptr, nullptr, lengths, plan,
             0, nullptr, B, false, (cudaStream_t)stream};
  const int e = launch_path_plan(c);
  return e ? cuda_fail(e, w) : ABRB_OK;
}

static int path_fill(const abrb_path_params *p, const double *table, const double *start, const double *target,
                     const double *v0, const double *v1, const double *so, const double *to, const abrb_path_rec *plan,
                     const int64_t *lengths, int64_t s_max, void *path, int64_t B, void *stream, bool f32) {
  const char *w = f32 ? "abrb_path_fill_f32" : "abrb_path_fill_f64";
  int rc = path_check(w, p, table, start, target, v0, v1, B);
  if (rc) return rc;
  if (s_max < 0 || s_max > (int64_t(1) << 30)) return fail(ABRB_EINVAL, std::string(w) + ": s_max outside 0 .. 2^30");
  if ((so == nullptr) != (to == nullptr))
    return fail(ABRB_EINVAL, std::string(w) + ": give both orientations or neither");
  if (B == 0 || s_max == 0) return ABRB_OK;
  const void *ptrs[] = {plan, lengths, so, to};
  for (int i = 0; i < 4; ++i) {
    if (!ptrs[i] && i < 2) return fail(ABRB_EINVAL, std::string(w) + ": NULL argument");
    if (ptrs[i] && !aligned_elem(ptrs[i], false)) return fail(ABRB_EINVAL, std::string(w) + ": misaligned pointer");
  }
  if (!path) return fail(ABRB_EINVAL, std::string(w) + ": NULL argument");
  if (!aligned_elem(path, f32)) return fail(ABRB_EINVAL, std::string(w) + ": misaligned pointer");
  if ((rc = ensure_device())) return rc;
  PathCall c{*p, table, start, target, nullptr, v0, v1, so, to, const_cast<int64_t *>(lengths),
             const_cast<abrb_path_rec *>(plan), s_max, path, B, f32, (cudaStream_t)stream};
  const int e = launch_path_fill(c);
  return e ? cuda_fail(e, w) : ABRB_OK;
}

int abrb_path_fill_f64(const abrb_path_params *p, const double *table, const double *start, const double *target,
                       const double *start_velocity, const double *target_velocity, const double *start_orientation,
                       const double *target_orientation, const abrb_path_rec *plan, const int64_t *lengths,
                       int64_t s_max, double *path, int64_t B, void *stream) {
  return path_fill(p, table, start, target, start_velocity, target_velocity, start_orientation, target_orientation,
                   plan, lengths, s_max, path, B, stream, false);
}
int abrb_path_fill_f32(const abrb_path_params *p, const double *table, const double *start, const double *target,
                       const double *start_velocity, const double *target_velocity, const double *start_orientation,
                       const double *target_orientation, const abrb_path_rec *plan, const int64_t *lengths,
                       int64_t s_max, float *path, int64_t B, void *stream) {
  return path_fill(p, table, start, target, start_velocity, target_velocity, start_orientation, target_orientation,
                   plan, lengths, s_max, path, B, stream, true);
}

}  // extern "C"
