// TEST INFRASTRUCTURE ONLY — never loaded by the abr_control_b200 package.
// The path planner's per-row and per-step functions (abrb_path.cuh) on the CPU: phase 1's plan_row with the warp's
// summation order replayed (HostSum), and the rows of phase 2 from the same per-step functions, with sequential
// cumulative sums in place of the CTA's scans.
#include "../../abr_control_b200/csrc/abrb_path.cuh"

#include <vector>

using namespace abrb;

extern "C" {

int64_t pl_plan_row(const abrb_path_params *p, const double *table, const double *start, const double *target,
                    double vmax, double v0, double v1, abrb_path_rec *rec) {
  return path::plan_row(*p, table, start, target, vmax, v0, v1, *rec, path::HostSum{});
}

// rows (S, w) of one planned path, w = 12 if so and to are given, else 6
int pl_fill_row(const abrb_path_params *p, const double *table, const double *start, const double *target, double v0,
                double v1, const double *so, const double *to, const abrb_path_rec *rec, int S, double *out) {
  path::Frame F;
  if (path::frame_of(start, target, F)) return -1;
  const int P = p->n_points;
  std::vector<double> arc(P), xyz(3 * P), ps(S);
  arc[0] = 0.0;
  for (int i = 0; i < P; ++i) {
    if (i > 0) arc[i] = arc[i - 1] + path::seg_len(F, table, i);
    path::warp_point(F, table, i, &xyz[3 * i]);
  }
  const path::Profile Pr = path::profile_of(*p, *rec, v0, v1);
  double acc = 0.0;
  for (int k = 0; k < S; ++k) ps[k] = acc = acc + path::step_at(Pr, k);
  const int w = so ? 12 : 6;
  std::vector<double> pos(3 * S), eul(3 * S);
  for (int k = 0; k < S; ++k) path::interp(arc.data(), xyz.data(), P, ps[k], &pos[3 * k]);
  if (so) {
    double q0[4], q1[4];
    path::unit_quat(so, p->axes, q0);
    path::unit_quat(to, p->axes, q1);
    for (int k = 0; k < S; ++k) path::orient_at(q0, q1, p->axes, &pos[0], &pos[3 * (S - 1)], &pos[3 * k], &eul[3 * k]);
  }
  for (int k = 0; k < S; ++k) {
    const int km = k > 0 ? k - 1 : k, kp = k < S - 1 ? k + 1 : k;
    for (int c = 0; c < 3; ++c) {
      out[k * w + c] = pos[3 * k + c];
      out[k * w + 3 + c] = path::gradient_at(pos[3 * km + c], pos[3 * k + c], pos[3 * kp + c], k, S, p->dt);
      if (so) {
        out[k * w + 6 + c] = eul[3 * k + c];
        out[k * w + 9 + c] = path::gradient_at(eul[3 * km + c], eul[3 * k + c], eul[3 * kp + c], k, S, p->dt);
      }
    }
  }
  return 0;
}

// vel_profile.generate(va, vb) of n samples
void pl_ramp(const abrb_path_params *p, double va, double vb, int n, double *out) {
  const path::Ramp r = path::ramp_make(*p, va, vb, n);
  for (int k = 0; k < n; ++k) out[k] = path::ramp_at(r, k);
}

void pl_quat_from_euler(const double *e, const int32_t *axes, double *q) {
  path::quat_from_euler(e[0], e[1], e[2], axes, q);
}

void pl_euler_from_quat(const double *q, const int32_t *axes, double *e) { path::euler_from_quat(q, axes, e); }

void pl_slerp(const double *q0, const double *q1, double f, double *out) { path::slerp(q0, q1, f, out); }
}
