// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// hostsim.cpp plus the choice between the plain and the general OSC instantiation (osc_plain, abrb_host.hpp): runs
// osc_state with the instantiation the library's kernels pick for a call (osc_go / rollout_go, kernels.cu), or the
// general one on request, so that `pytest -m "not gpu"` checks the plain path against the oracle and the general path.
#include "hostsim.cpp"

namespace {

template <typename T, int N, bool ORTHO>
void osc_pick_loop(const ChainHost &h, const abrb_osc_params &p, int frame, const double *xoff, const double *q,
                   const double *dq, const double *target, const double *tv, int64_t B, double *u, double *train,
                   double *ddq, double *ierr, bool allow_plain) {
  ChainK<T, N> P;
  fill_chain<T, N>(h, P);
  OscK<T, N> O;
  fill_osc<T, N>(p, frame, xoff, O);
  const bool kd6 = (O.dof_mask & 56u) != 0;
  const bool plain = allow_plain && osc_plain(p, N, frame, kd6 ? 6 : 3, tv != nullptr, ierr != nullptr);
  for (int64_t b = 0; b < B; ++b) {
    T qq[N], dd[N], tg[6], tvv[6], uu[N], tr[N], acc[N], ie[6];
    for (int k = 0; k < N; ++k) {
      qq[k] = T(q[b * N + k]);
      dd[k] = T(dq[b * N + k]);
    }
    for (int c = 0; c < 6; ++c) {
      tg[c] = T(target[b * 6 + c]);
      tvv[c] = tv ? T(tv[b * 6 + c]) : T(0);
      ie[c] = ierr ? T(ierr[b * 6 + c]) : T(0);
    }
    const T *tvp = tv ? tvv : nullptr;
    T *iep = ierr ? ie : nullptr;
    Kin<T, N, ORTHO> K;
    if (kd6) {
      if (plain)
        osc_state<T, N, 6, true, true>(P, O, qq, dd, tg, tvp, iep, uu, tr, acc, K);
      else
        osc_state<T, N, 6, true, false>(P, O, qq, dd, tg, tvp, iep, uu, tr, acc, K);
    } else {
      if (plain)
        osc_state<T, N, 3, true, true>(P, O, qq, dd, tg, tvp, iep, uu, tr, acc, K);
      else
        osc_state<T, N, 3, true, false>(P, O, qq, dd, tg, tvp, iep, uu, tr, acc, K);
    }
    for (int c = 0; c < 6; ++c)
      if (ierr) ierr[b * 6 + c] = double(ie[c]);
    for (int k = 0; k < N; ++k) {
      u[b * N + k] = double(uu[k]);
      if (train) train[b * N + k] = double(tr[k]);
      if (ddq) ddq[b * N + k] = double(acc[k]);
    }
  }
}

}  // namespace

extern "C" {

// target, tv: (B, 6).  general != 0 runs the general instantiation even for calls that qualify for the plain one.
int ps_osc(const abrb_chain_desc *d, const abrb_osc_params *p, int f32, int general, int frame, const double *xoff,
           const double *q, const double *dq, const double *target, const double *tv, int64_t B, double *u,
           double *train, double *ddq, double *ierr) {
  ChainHost h;
  if (!chain_from_desc(*d, h).empty()) return ABRB_EINVAL;
  if (!check_osc(h.n, *p).empty()) return ABRB_EUNSUP;
  if ((p->ki != 0.0) != (ierr != nullptr)) return ABRB_EINVAL;
  const bool ortho = h.ortho;
  DISPATCH_N(osc_pick_loop, h, *p, frame, xoff, q, dq, target, tv, B, u, train, ddq, ierr, general == 0);
  return 0;
}

// 1 if a call with these parameters runs the plain OSC instantiation
int ps_osc_plain(const abrb_osc_params *p, int n, int frame, int has_tv, int has_ierr) {
  const bool kd6 = p->ctrlr_dof[3] || p->ctrlr_dof[4] || p->ctrlr_dof[5];
  return osc_plain(*p, n, frame, kd6 ? 6 : 3, has_tv != 0, has_ierr != 0) ? 1 : 0;
}
}
