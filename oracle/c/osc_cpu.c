/*
 * TEST / BASELINE INFRASTRUCTURE — not part of the product (libabrb.so never links or loads this).
 *
 * CPU restatement in plain C of the NumPy half of the reference's OSC path, so that the reference's CPU
 * implementation can be timed without the Python interpreter in the loop:
 *   OSC._Mx                     /root/reference/abr_control/controllers/osc.py:120-147
 *   OSC._calc_orientation_forces osc.py:149-196  (+ utils/transformations.py:1096-1147, 1192-1302)
 *   OSC._velocity_limiting      osc.py:198-215
 *   OSC.generate                osc.py:217-320
 *   Damping / RestingConfig     controllers/damping.py:21-32, resting_config.py:25-42 + joint.py:104-131
 * numpy.linalg.{inv,det,pinv,eigh} (LAPACK in the reference) are restated as Gauss-Jordan with partial
 * pivoting and cyclic Jacobi; results agree with the NumPy oracle (oracle/osc_oracle.py) to rounding, which
 * tests/test_oracle_golden.py::test_c_restatement_vs_numpy_oracle checks on the golden cases.
 *
 * The rigid-body quantities J, M, g, C, Tx, R are INPUTS here: either produced by the reference's own
 * generated C (oracle/_ref, see ref_ur5_driver.c — cpu_baseline kind "reference") or by the NumPy oracle.
 */
#include <math.h>
#include <string.h>

#define NMAX 8

typedef struct osc_cfg {
  int n;                 /* joints */
  double kp, ko, kv;
  int use_vmax;
  double vmax[2];
  int dof[6];
  int use_g, use_C, alg;
  double damp_kv;        /* < 0: no Damping null controller */
  int use_rest;          /* RestingConfig */
  double rest_kp, rest_kv, rest[NMAX];
  int rest_mask[NMAX];
} osc_cfg;

/* ---- small dense helpers (row-major, leading dimension = n) ------------------------------------ */
static int gauss_jordan_inv(int n, const double *A, double *Ainv, double *det_out) {
  double a[NMAX * 2 * NMAX];
  double det = 1.0;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) {
      a[i * 2 * n + j] = A[i * n + j];
      a[i * 2 * n + n + j] = i == j ? 1.0 : 0.0;
    }
  for (int c = 0; c < n; ++c) {
    int p = c;
    for (int r = c + 1; r < n; ++r)
      if (fabs(a[r * 2 * n + c]) > fabs(a[p * 2 * n + c])) p = r;
    if (p != c) {
      for (int j = 0; j < 2 * n; ++j) {
        double t = a[c * 2 * n + j];
        a[c * 2 * n + j] = a[p * 2 * n + j];
        a[p * 2 * n + j] = t;
      }
      det = -det;
    }
    const double piv = a[c * 2 * n + c];
    det *= piv;
    if (piv == 0.0) {
      if (det_out) *det_out = 0.0;
      return -1;
    }
    const double ip = 1.0 / piv;
    for (int j = 0; j < 2 * n; ++j) a[c * 2 * n + j] *= ip;
    for (int r = 0; r < n; ++r)
      if (r != c) {
        const double f = a[r * 2 * n + c];
        if (f != 0.0)
          for (int j = 0; j < 2 * n; ++j) a[r * 2 * n + j] -= f * a[c * 2 * n + j];
      }
  }
  if (Ainv)
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) Ainv[i * n + j] = a[i * 2 * n + n + j];
  if (det_out) *det_out = det;
  return 0;
}

/* symmetric eigen-decomposition, cyclic Jacobi: A = V diag(w) V^T */
static void jacobi_eigh(int n, const double *Ain, double *w, double *V) {
  double A[NMAX * NMAX];
  memcpy(A, Ain, sizeof(double) * n * n);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) V[i * n + j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < n; ++i) {
      diag += A[i * n + i] * A[i * n + i];
      for (int j = i + 1; j < n; ++j) off += A[i * n + j] * A[i * n + j];
    }
    if (off <= 1e-32 * diag || off == 0.0) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[p * n + q];
        if (apq == 0.0) continue;
        const double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq;
          A[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk;
          A[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq;
          V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}

/* numpy.linalg.pinv(A, rcond) for symmetric A: drop |eigenvalue| <= rcond * max|eigenvalue| */
static void pinv_sym(int n, const double *A, double rcond, double *P) {
  double w[NMAX], V[NMAX * NMAX];
  jacobi_eigh(n, A, w, V);
  double lmax = 0;
  for (int i = 0; i < n; ++i)
    if (fabs(w[i]) > lmax) lmax = fabs(w[i]);
  for (int i = 0; i < n * n; ++i) P[i] = 0.0;
  for (int e = 0; e < n; ++e) {
    if (!(fabs(w[e]) > rcond * lmax)) continue;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) P[i * n + j] += V[i * n + e] * V[j * n + e] / w[e];
  }
}

/* utils/transformations.py:1192-1271 (isprecise=False): eigenvector of the largest eigenvalue of K/3 */
static void quat_from_matrix(const double *m /*3x3*/, double *q) {
  double K[16] = {0}, w[4], V[16];
  K[0] = m[0] - m[4] - m[8];
  K[5] = m[4] - m[0] - m[8];
  K[10] = m[8] - m[0] - m[4];
  K[15] = m[0] + m[4] + m[8];
  K[4] = K[1] = m[1] + m[3];
  K[8] = K[2] = m[2] + m[6];
  K[9] = K[6] = m[5] + m[7];
  K[12] = K[3] = m[7] - m[5];
  K[13] = K[7] = m[2] - m[6];
  K[14] = K[11] = m[3] - m[1];
  for (int i = 0; i < 16; ++i) K[i] /= 3.0;
  jacobi_eigh(4, K, w, V);
  int b = 0;
  for (int i = 1; i < 4; ++i)
    if (w[i] > w[b]) b = i;
  q[0] = V[3 * 4 + b];
  q[1] = V[0 * 4 + b];
  q[2] = V[1 * 4 + b];
  q[3] = V[2 * 4 + b];
  if (q[0] < 0.0)
    for (int i = 0; i < 4; ++i) q[i] = -q[i];
  const double nn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; ++i) q[i] /= nn;
}

static void quat_from_euler_rxyz(double al, double be, double ga, double *q) { /* transformations.py:1096-1147 */
  const double ai = ga / 2.0, aj = -be / 2.0, ak = al / 2.0; /* frame=1 swaps, parity=1 negates aj */
  const double ci = cos(ai), si = sin(ai), cj = cos(aj), sj = sin(aj), ck = cos(ak), sk = sin(ak);
  const double cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  q[0] = cj * cc + sj * ss;
  q[3] = cj * sc - sj * cs;
  q[2] = -(cj * ss + sj * cc);
  q[1] = cj * cs - sj * sc;
  const double nn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; ++i) q[i] /= nn;
}

static void euler_matrix_rxyz(double al, double be, double ga, double *R) { /* transformations.py:973-1035 */
  const double ai = -ga, aj = -be, ak = -al;
  const double si = sin(ai), sj = sin(aj), sk = sin(ak), ci = cos(ai), cj = cos(aj), ck = cos(ak);
  const double cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  R[8] = cj * ck;
  R[7] = sj * sc - cs;
  R[6] = sj * cc + ss;
  R[5] = cj * sk;
  R[4] = sj * ss + cc;
  R[3] = sj * cs - sc;
  R[2] = -sj;
  R[1] = cj * si;
  R[0] = cj * ci;
}

static double wrap_pm_pi(double d) {
  const double two_pi = 2.0 * M_PI;
  double r = fmod(d + M_PI, two_pi);
  if (r < 0) r += two_pi;
  return r - M_PI;
}

/* One OSC.generate from already-evaluated rigid-body quantities (all fp64, row-major):
 * J[6][n], M[n][n], g[n], Cm[n][n] (may be NULL unless use_C), x[3] = Tx(ref_frame), R[3][3]. */
void osc_from_quantities(const osc_cfg *c, const double *J6, const double *M, const double *g, const double *Cm,
                         const double *x, const double *R, const double *q, const double *dq, const double *target,
                         const double *tv, double *u, double *train) {
  const int n = c->n;
  int idx[6], k = 0;
  for (int r = 0; r < 6; ++r)
    if (c->dof[r]) idx[k++] = r;
  double J[6 * NMAX], Minv[NMAX * NMAX], JM[6 * NMAX], S[36], Mx[36];
  for (int a = 0; a < k; ++a)
    for (int j = 0; j < n; ++j) J[a * n + j] = J6[idx[a] * n + j];
  gauss_jordan_inv(n, M, Minv, 0);
  for (int a = 0; a < k; ++a)
    for (int j = 0; j < n; ++j) {
      double s = 0;
      for (int i = 0; i < n; ++i) s += J[a * n + i] * Minv[i * n + j];
      JM[a * n + j] = s;
    }
  for (int a = 0; a < k; ++a)
    for (int b = 0; b < k; ++b) {
      double s = 0;
      for (int i = 0; i < n; ++i) s += JM[a * n + i] * J[b * n + i];
      S[a * k + b] = s;
    }
  double det = 0;
  if (gauss_jordan_inv(k, S, Mx, &det) != 0 || !(fabs(det) >= 1e-3)) {
    /* symmetrise rounding noise before the eigen route (S is symmetric in exact arithmetic) */
    double Ss[36];
    for (int a = 0; a < k; ++a)
      for (int b = 0; b < k; ++b) Ss[a * k + b] = 0.5 * (S[a * k + b] + S[b * k + a]);
    pinv_sym(k, Ss, 1e-3 * 0.1, Mx);
  }
  double e[6] = {0, 0, 0, 0, 0, 0};
  if (c->dof[0] || c->dof[1] || c->dof[2])
    for (int i = 0; i < 3; ++i) e[i] = x[i] - target[i];
  if (c->dof[3] || c->dof[4] || c->dof[5]) {
    if (c->alg == 0) {
      double qd[4], qe[4], qr[4];
      quat_from_euler_rxyz(target[3], target[4], target[5], qd);
      quat_from_matrix(R, qe);
      qe[1] = -qe[1];
      qe[2] = -qe[2];
      qe[3] = -qe[3];
      qr[0] = -qd[1] * qe[1] - qd[2] * qe[2] - qd[3] * qe[3] + qd[0] * qe[0];
      qr[1] = qd[1] * qe[0] + qd[2] * qe[3] - qd[3] * qe[2] + qd[0] * qe[1];
      qr[2] = -qd[1] * qe[3] + qd[2] * qe[0] + qd[3] * qe[1] + qd[0] * qe[2];
      qr[3] = qd[1] * qe[2] - qd[2] * qe[1] + qd[3] * qe[0] + qd[0] * qe[3];
      const double sg = qr[0] > 0 ? 1.0 : (qr[0] < 0 ? -1.0 : 0.0);
      for (int i = 0; i < 3; ++i) e[3 + i] = -qr[1 + i] * sg;
    } else {
      double Rd[9], Red[9], qed[4];
      euler_matrix_rxyz(target[3], target[4], target[5], Rd);
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) Red[a * 3 + b] = R[0 * 3 + a] * Rd[0 * 3 + b] + R[1 * 3 + a] * Rd[1 * 3 + b] + R[2 * 3 + a] * Rd[2 * 3 + b];
      quat_from_matrix(Red, qed);
      for (int a = 0; a < 3; ++a) e[3 + a] = -(R[a * 3 + 0] * qed[1] + R[a * 3 + 1] * qed[2] + R[a * 3 + 2] * qed[3]);
    }
  }
  if (c->use_vmax) {
    const double lx = c->vmax[0] / c->kp * c->kv, la = c->vmax[1] / c->ko * c->kv;
    const double nx = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), na = sqrt(e[3] * e[3] + e[4] * e[4] + e[5] * e[5]);
    const double sx = nx > lx ? lx / nx : 1.0, sa = na > la ? la / na : 1.0;
    for (int i = 0; i < 3; ++i) {
      e[i] = c->kv * sx * (c->kp / c->kv) * e[i];
      e[3 + i] = c->kv * sa * (c->ko / c->kv) * e[3 + i];
    }
  } else {
    for (int i = 0; i < 3; ++i) {
      e[i] *= c->kp;
      e[3 + i] *= c->ko;
    }
  }
  int tv_zero = 1;
  if (tv)
    for (int i = 0; i < 6; ++i)
      if (tv[i] != 0.0) tv_zero = 0;
  for (int i = 0; i < n; ++i) {
    double s = 0;
    if (tv_zero)
      for (int j = 0; j < n; ++j) s += M[i * n + j] * dq[j];
    u[i] = tv_zero ? -c->kv * s : 0.0;
  }
  if (!tv_zero) {
    double dx[6] = {0, 0, 0, 0, 0, 0};
    for (int a = 0; a < k; ++a) {
      double s = 0;
      for (int j = 0; j < n; ++j) s += J[a * n + j] * dq[j];
      dx[idx[a]] = s;
    }
    for (int i = 0; i < 6; ++i) e[i] += c->kv * (dx[i] - tv[i]);
  }
  double y[6], f[6];
  for (int a = 0; a < k; ++a) y[a] = e[idx[a]];
  for (int a = 0; a < k; ++a) {
    double s = 0;
    for (int b = 0; b < k; ++b) s += Mx[a * k + b] * y[b];
    f[a] = s;
  }
  for (int i = 0; i < n; ++i) {
    double s = 0;
    for (int a = 0; a < k; ++a) s += J[a * n + i] * f[a];
    u[i] -= s;
  }
  if (c->use_C)
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int j = 0; j < n; ++j) s += Cm[i * n + j] * dq[j];
      u[i] -= s;
    }
  if (train)
    for (int i = 0; i < n; ++i) train[i] = u[i];
  if (c->use_g)
    for (int i = 0; i < n; ++i) u[i] -= g[i];
  const int n_null = (c->damp_kv >= 0 ? 1 : 0) + (c->use_rest ? 1 : 0);
  for (int nc = 0; nc < n_null; ++nc) {
    double wv[NMAX], un[NMAX], t1[6], t2[6];
    const int is_damp = (c->damp_kv >= 0) && nc == 0;
    for (int j = 0; j < n; ++j) {
      if (is_damp) {
        wv[j] = -c->damp_kv * dq[j];
      } else {
        const double qt = c->rest_mask[j] ? wrap_pm_pi(c->rest[j] - q[j]) : 0.0;
        wv[j] = c->rest_kp * qt + c->rest_kv * (0.0 - dq[j]);
      }
    }
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int j = 0; j < n; ++j) s += M[i * n + j] * wv[j];
      un[i] = s;
    }
    /* u += (I - J^T (M^-1 J^T Mx)^T) u_null = u_null - J^T Mx^T J M^-1 u_null */
    for (int a = 0; a < k; ++a) {
      double s = 0;
      for (int j = 0; j < n; ++j) s += JM[a * n + j] * un[j];
      t1[a] = s;
    }
    for (int a = 0; a < k; ++a) {
      double s = 0;
      for (int b = 0; b < k; ++b) s += Mx[b * k + a] * t1[b];
      t2[a] = s;
    }
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int a = 0; a < k; ++a) s += J[a * n + i] * t2[a];
      u[i] += un[i] - s;
    }
  }
}

/* batch wrapper over precomputed quantities (used by tests/test_oracle_golden.py::test_c_restatement_vs_numpy_oracle
   and tests/test_gpu_fullsize.py) */
void osc_from_quantities_batch(const osc_cfg *c, long B, const double *J6, const double *M, const double *g,
                               const double *Cm, const double *x, const double *R, const double *q, const double *dq,
                               const double *target, const double *tv, double *u, double *train) {
  const int n = c->n;
  for (long b = 0; b < B; ++b)
    osc_from_quantities(c, J6 + b * 6 * n, M + b * n * n, g + b * n, Cm ? Cm + b * n * n : 0, x + b * 3, R + b * 9,
                        q + b * n, dq + b * n, target + b * 6, tv ? tv + b * 6 : 0, u + b * n,
                        train ? train + b * n : 0);
}
