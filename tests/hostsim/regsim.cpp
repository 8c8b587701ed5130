// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// plantsim.cpp plus the inverse-dynamics regressor: runs inverse_dynamics_regressor (abrb_regress.cuh), the per-state
// body of regressor_kernel, with the halves of each record placed at the offsets the kernel stores them to, so that
// `pytest -m "not gpu"` checks it against the oracle and against inverse_dynamics_state (pl_dynamics, kind 1).
#include "plantsim.cpp"

#include "../../abr_control_b200/csrc/abrb_regress.cuh"

namespace {

template <typename T, int N>
struct RegSink {  // receives each finished half of a state's (6N, N) record
  double *rec;
  template <int LEN>
  void put(int off, const T *half) {
    for (int i = 0; i < LEN; ++i) rec[off + i] = double(half[i]);
  }
};

template <typename T, int N, bool ORTHO>
void regressor_loop(const ChainHost &h, const double *gravity, const double *q, const double *dq, const double *ddq,
                    int64_t B, double *Yt) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  T grav[6];
  for (int c = 0; c < 6; ++c) grav[c] = T(gravity[c]);
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], aa[N];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
      aa[k] = T(ddq[b * N + k]);
    }
    RegSink<T, N> sink{Yt + b * RegressorLayout<N>::kRecord};
    Kin<T, N, ORTHO> K;
    inverse_dynamics_regressor<T, N>(P, grav, qq, dd, aa, sink, K);
  }
}

}  // namespace

extern "C" {

// Yt: (B, 6n, n), element (b, p, a) = d u_a / d theta_p of state b
int rs_regressor(const abrb_chain_desc *d, int f32, const double *q, const double *dq, const double *ddq, int64_t B,
                 double *Yt) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  const bool ortho = h.ortho;
  DISPATCH_N(regressor_loop, h, d->gravity, q, dq, ddq, B, Yt);
  return 0;
}
}
