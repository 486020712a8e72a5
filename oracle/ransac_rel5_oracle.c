/* oracle/ransac_rel5_oracle.c — CPU restatement of the central relative-pose (5-point) RANSAC of
 * RelNonCentralPosSolver::computePose (RelNonCentralPosSolver.cpp:343-377) from caller-supplied samples.
 * TEST INFRASTRUCTURE ONLY (tests/, tools/); never linked into covins_b200/.  It is the bit-for-bit reference of
 * cvb_ransac_central_relative_pose_batch (covins_b200/csrc/ransac_rel.cu, ransac_rel_kernel<Solver5>).
 * It includes the 17-point restatement (ransac_rel_oracle.c, unchanged) for its helpers: the per-correspondence score
 * rel_score, the camera-pair model pair_model and the 3x3 inverse.  A central problem is scored as the kernel scores it: the
 * camera-pair model of one identity camera per side, then rel_score.
 * Only + - * / and sqrt, fixed iteration counts; plain IEEE double without contraction (compile with -ffp-contract=off).
 */
#include "ransac_rel_oracle.c"

/* one central problem's correspondences */
typedef struct {
  int n;
  const double *f1, *f2, *s1, *s2;
} rel5_problem;

/* the score's triangulation (opengv::triangulation::triangulate2; the same operations as the first half of rel_score) of
 * bearings a (view 1), bb (view 2) under P = [R12|t12], ti = -R12^T t12: X in view 1, r2 = R12^T X + ti in view 2 */
static void rel5_triangulate(const double* M, const double* ti, const double* a, const double* bb, double* X, double* r2) {
  const double t[3] = {M[3], M[7], M[11]};
  double u[3];
  for (int r = 0; r < 3; r++) u[r] = (M[4 * r] * bb[0] + M[4 * r + 1] * bb[1]) + M[4 * r + 2] * bb[2];
  const double b0 = (t[0] * a[0] + t[1] * a[1]) + t[2] * a[2], b1 = (t[0] * u[0] + t[1] * u[1]) + t[2] * u[2];
  const double A00 = (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2], A10 = (a[0] * u[0] + a[1] * u[1]) + a[2] * u[2];
  const double A01 = -A10, A11 = -((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]);
  const double det = A00 * A11 - A01 * A10;
  const double l0 = (A11 * b0 - A01 * b1) / det, l1 = (A00 * b1 - A10 * b0) / det;
  for (int r = 0; r < 3; r++) X[r] = (l0 * a[r] + (t[r] + l1 * u[r])) / 2.0;
  for (int r = 0; r < 3; r++) r2[r] = ((M[r] * X[0] + M[4 + r] * X[1]) + M[8 + r] * X[2]) + ti[r];
}

/* ---- the 5-point hypothesis ----
 * ASSUMPTIONS (opengv is not in the tree):
 *   [N] Stewénius' eigen-decomposition is replaced by Nistér's degree-10 polynomial; only its real roots are kept, where
 *       opengv takes the real parts of all ten complex solutions.
 *   [T] |t| = 1, where opengv scales t by E's largest singular value; the score does not depend on |t|.
 *   [Q] CentralRelativePoseSacProblem::computeModelCoefficients' quality test runs on the sample's five points only.
 * Hypothesis:
 *   1. q_i = vec(f1_i f2_i^T) (row-major, q_i . vec(E) = f1^T E f2); Householder QR of Q^T (9x5) as rel17's, invalid if
 *      min |r_kk| < REL_RANK_TOL max |r_kk|; null-space basis X, Y, Z, W = H_0..H_4 e_5..e_8.
 *   2. E = xX + yY + zZ + W, E_ij the linear polynomial (X_ij, Y_ij, Z_ij, W_ij) in (x, y, z, 1).  Rows 0-8 of the 10x20
 *      matrix: entry (r, c) row-major of 2 E E^T E - tr(E E^T) E, with S_rk = sum_m E_rm E_km, tr = (S_00 + S_11) + S_22,
 *      row = 2 (sum_k S_rk E_kc) - tr E_rc; row 9: det E = E_00 M_0 + E_01 M_1 + E_02 M_2 (M_0 = E_11 E_22 - E_12 E_21,
 *      M_1 = E_12 E_20 - E_10 E_22, M_2 = E_10 E_21 - E_11 E_20).  Every product goes through rel5_pmul, columns in Nistér's
 *      monomial order (x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy xz^2 xz x yz^2 yz y z^3 z^2 z 1).
 *   3. Gauss-Jordan on the left 10x10 block, partial pivoting (largest |value|, first row on ties), invalid if a pivot is
 *      below REL5_PIVOT_TOL times the largest |entry| of the matrix.  B(z) rows <e> - z<f>, <g> - z<h>, <i> - z<j> (rows 4-9);
 *      n(z) = det B(z) (degree 10) by cofactors along row 0.  Real roots: with the Cauchy bound b = 1 + max |n_i / n_10|
 *      (invalid if not finite), the roots of n^(d) for d = 9, 8, ..., 0 in turn, each one per sign change of n^(d) between
 *      consecutive roots of n^(d+1) (and -b, b): REL5_BISECT bisection steps, then REL5_NEWTON Newton steps each kept only
 *      inside the final bracket.  Per root, ascending: (x, y, 1) ~ the largest of the three cross products of B(z)'s rows
 *      (first on ties), then rel5_polish: Gauss-Newton steps on the unreduced cubics, which recover the digits the elimination
 *      and the degree-10 polynomial lose on ill-conditioned samples.
 *   4. E scaled to tr(E E^T) / 2 = 1; b = the largest of E's three column cross products (first on ties), normalised;
 *      R_+- = cof(E) -+ [b]x E; candidates (R_+, b), (R_+, -b), (R_-, b), (R_-, -b).
 *   5. quality = sum over the sample's points in order of (1 - f1 . X/|X|) + (1 - f2 . r2/|r2|), X and r2 from the score's
 *      triangulation; the strictly lowest finite quality over roots x candidates wins; no finite one: invalid. */
#define REL5_SAMPLE 5
#define REL5_PIVOT_TOL 1e-10
enum { REL5_BISECT = 64, REL5_NEWTON = 4, REL5_POLISH = 6 };

/* products of polynomials linear in (x, y, z): linear terms (x, y, z, 1); quadratic terms (x^2, xy, xz, x, y^2, yz, y, z^2, z, 1);
 * cubic terms in Nistér's order.  rel5_qidx / rel5_cidx: index of (quadratic or linear term i) x (linear term j) */
static const int rel5_qidx[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
static const int rel5_cidx[10][4] = {{0, 2, 4, 5}, {2, 3, 8, 9}, {4, 8, 10, 11}, {5, 9, 11, 12}, {3, 1, 6, 7},
                                     {8, 6, 13, 14}, {9, 7, 14, 15}, {10, 13, 16, 17}, {11, 14, 17, 18}, {12, 15, 18, 19}};
/* out += p * l, p of np terms, term i times linear term j into out[idx[i][j]], i outer, j inner */
static void rel5_pmul(const double* p, int np, const int (*idx)[4], const double* l, double* out) {
  for (int i = 0; i < np; i++)
    for (int j = 0; j < 4; j++) out[idx[i][j]] = out[idx[i][j]] + p[i] * l[j];
}
/* out (ascending powers of z) += a (na coefficients) * b (nb coefficients), i outer, j inner */
static void rel5_upmul(const double* a, int na, const double* b, int nb, double* out) {
  for (int i = 0; i < na; i++)
    for (int j = 0; j < nb; j++) out[i + j] = out[i + j] + a[i] * b[j];
}
static double rel5_horner(const double* c, int d, double x) {
  double v = c[d];
  for (int i = d - 1; i >= 0; i--) v = v * x + c[i];
  return v;
}
static int rel5_sign(double v) { return (v > 0.0) - (v < 0.0); }
/* the root of c (degree d, derivative dc) in [a, b] if c changes sign there (c(a) != 0, c(b) = 0 counts); returns found */
static int rel5_root(const double* c, int d, const double* dc, double a, double b, double* root) {
  const int sa = rel5_sign(rel5_horner(c, d, a)), sb = rel5_sign(rel5_horner(c, d, b));
  if (sa == 0 || sb == sa) return 0;
  for (int it = 0; it < REL5_BISECT; it++) {
    const double m = 0.5 * a + 0.5 * b;
    if (rel5_sign(rel5_horner(c, d, m)) == sa) a = m; else b = m;
  }
  double x = 0.5 * a + 0.5 * b;
  for (int it = 0; it < REL5_NEWTON; it++) {
    const double xn = x - rel5_horner(c, d, x) / rel5_horner(dc, d - 1, x);
    if (xn >= a && xn <= b) x = xn;
  }
  *root = x;
  return 1;
}
static void rel5_cross_max(const double* r0, const double* r1, const double* r2, double* v, double* nv) {
  double c[3][3];
  cross3(r0, r1, c[0]); cross3(r0, r2, c[1]); cross3(r1, r2, c[2]);
  int k = 0;
  double best = dot3(c[0], c[0]);
  for (int j = 1; j < 3; j++) {
    const double nj = dot3(c[j], c[j]);
    if (nj > best) { best = nj; k = j; }
  }
  memcpy(v, c[k], 24);
  *nv = best;
}

/* exponents (x, y, z) of the cubic terms in Nistér's order */
static const int rel5_exp[20][3] = {{3, 0, 0}, {0, 3, 0}, {2, 1, 0}, {1, 2, 0}, {2, 0, 1}, {2, 0, 0}, {0, 2, 1}, {0, 2, 0}, {1, 1, 1}, {1, 1, 0},
                                    {1, 0, 2}, {1, 0, 1}, {1, 0, 0}, {0, 1, 2}, {0, 1, 1}, {0, 1, 0}, {0, 0, 3}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};
/* at most REL5_POLISH Gauss-Newton steps on the ten cubics A0 m(x, y, z) = 0 from v = (x, y, z): J^T J d = J^T F by inv3,
 * v -= d; the first step that does not lower |F|^2 (or leaves the finite range) is undone and ends the polish */
static void rel5_polish(const double (*A0)[20], double* v) {
  double prev[3] = {v[0], v[1], v[2]}, rprev = INFINITY;
  for (int it = 0; it <= REL5_POLISH; it++) {
    double pw[3][4], m[4][20];   /* m[0] = monomials, m[1..3] = their partial derivatives in x, y, z */
    for (int a = 0; a < 3; a++) {
      pw[a][0] = 1.0;
      for (int e = 1; e < 4; e++) pw[a][e] = pw[a][e - 1] * v[a];
    }
    for (int i = 0; i < 20; i++) {
      const int* ex = rel5_exp[i];
      m[0][i] = (pw[0][ex[0]] * pw[1][ex[1]]) * pw[2][ex[2]];
      for (int a = 0; a < 3; a++) {
        int e2[3] = {ex[0], ex[1], ex[2]};
        if (e2[a] == 0) { m[1 + a][i] = 0.0; continue; }
        e2[a]--;
        m[1 + a][i] = (((double)ex[a] * pw[0][e2[0]]) * pw[1][e2[1]]) * pw[2][e2[2]];
      }
    }
    double N[9], g[3], Ni[9], res = 0.0;
    for (int r = 0; r < 10; r++) {
      double F[4];
      for (int q = 0; q < 4; q++) {
        double acc = 0.0;
        for (int i = 0; i < 20; i++) acc = i == 0 ? A0[r][i] * m[q][i] : acc + A0[r][i] * m[q][i];
        F[q] = acc;
      }
      res = r == 0 ? F[0] * F[0] : res + F[0] * F[0];
      for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) N[3 * a + b] = r == 0 ? F[1 + a] * F[1 + b] : N[3 * a + b] + F[1 + a] * F[1 + b];
        g[a] = r == 0 ? F[1 + a] * F[0] : g[a] + F[1 + a] * F[0];
      }
    }
    if (!(res < rprev)) { memcpy(v, prev, 24); break; }
    if (it == REL5_POLISH) break;
    memcpy(prev, v, 24);
    rprev = res;
    inv3(N, Ni);
    for (int a = 0; a < 3; a++) v[a] = v[a] - ((Ni[3 * a] * g[0] + Ni[3 * a + 1] * g[1]) + Ni[3 * a + 2] * g[2]);
  }
}

/* per-sample intermediates for tests (nullable) */
typedef struct {
  int n_roots;
  double z[10], E[10][9], cand[10][4][12], quality[10][4];
} rel5_detail;

/* the hypothesis of the sample s[5] of a central problem (f1, f2, n); 0 = invalid */
static int rel5_hypothesis(const rel5_problem* P, const int32_t* s, double* model, rel5_detail* det) {
  if (det) det->n_roots = 0;
  if (P->n < REL5_SAMPLE) return 0;
  for (int i = 0; i < REL5_SAMPLE; i++)
    for (int j = i + 1; j < REL5_SAMPLE; j++)
      if (s[i] == s[j]) return 0;
  for (int i = 0; i < REL5_SAMPLE; i++)
    if (!finite_n(P->f1 + 3 * (size_t)s[i], 3) || !finite_n(P->f2 + 3 * (size_t)s[i], 3)) return 0;
  /* 1. null space of Q by the Householder QR of Q^T */
  double Qt[REL5_SAMPLE][9], alpha[REL5_SAMPLE], vtv[REL5_SAMPLE];
  for (int i = 0; i < REL5_SAMPLE; i++) {
    const double *a = P->f1 + 3 * (size_t)s[i], *b = P->f2 + 3 * (size_t)s[i];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) Qt[i][3 * r + c] = a[r] * b[c];
  }
  for (int k = 0; k < REL5_SAMPLE; k++) {
    double* col = Qt[k];
    double ss = 0.0;
    for (int i = k; i < 9; i++) ss = i == k ? col[i] * col[i] : ss + col[i] * col[i];
    const double sigma = sqrt(ss), ak = col[k];
    alpha[k] = ak >= 0.0 ? -sigma : sigma;
    col[k] = ak - alpha[k];
    vtv[k] = 2.0 * (ss + fabs(ak) * sigma);
    for (int j = k + 1; j < REL5_SAMPLE; j++) {
      double dot = 0.0;
      for (int i = k; i < 9; i++) dot = i == k ? col[i] * Qt[j][i] : dot + col[i] * Qt[j][i];
      const double c = (2.0 * dot) / vtv[k];
      for (int i = k; i < 9; i++) Qt[j][i] = Qt[j][i] - c * col[i];
    }
  }
  double rmax = 0.0;
  for (int k = 0; k < REL5_SAMPLE; k++) rmax = fabs(alpha[k]) > rmax ? fabs(alpha[k]) : rmax;
  int full_rank = rmax > 0.0;
  for (int k = 0; k < REL5_SAMPLE; k++)
    if (!(fabs(alpha[k]) >= REL_RANK_TOL * rmax)) full_rank = 0;
  if (!full_rank) return 0;
  double basis[4][9];   /* X, Y, Z, W */
  for (int j = 0; j < 4; j++) {
    double* x = basis[j];
    for (int i = 0; i < 9; i++) x[i] = i == REL5_SAMPLE + j ? 1.0 : 0.0;
    for (int k = REL5_SAMPLE - 1; k >= 0; k--) {
      double dot = 0.0;
      for (int i = k; i < 9; i++) dot = i == k ? Qt[k][i] * x[i] : dot + Qt[k][i] * x[i];
      const double c = (2.0 * dot) / vtv[k];
      for (int i = k; i < 9; i++) x[i] = x[i] - c * Qt[k][i];
    }
  }
  /* 2. the 10x20 coefficient matrix */
  double e[9][4], S[9][10], tr[10], A[10][20];
  for (int i = 0; i < 9; i++)
    for (int j = 0; j < 4; j++) e[i][j] = basis[j][i];
  for (int r = 0; r < 3; r++)
    for (int k = 0; k < 3; k++) {
      memset(S[3 * r + k], 0, sizeof(S[0]));
      for (int m = 0; m < 3; m++) rel5_pmul(e[3 * r + m], 4, rel5_qidx, e[3 * k + m], S[3 * r + k]);
    }
  for (int i = 0; i < 10; i++) tr[i] = (S[0][i] + S[4][i]) + S[8][i];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double Cc[20] = {0}, T[20] = {0};
      for (int k = 0; k < 3; k++) rel5_pmul(S[3 * r + k], 10, rel5_cidx, e[3 * k + c], Cc);
      rel5_pmul(tr, 10, rel5_cidx, e[3 * r + c], T);
      for (int m = 0; m < 20; m++) A[3 * r + c][m] = 2.0 * Cc[m] - T[m];
    }
  {
    static const int mi[3][4] = {{4, 8, 5, 7}, {5, 6, 3, 8}, {3, 7, 4, 6}};   /* M_c = E_a E_b - E_c' E_d' */
    double D[20] = {0};
    for (int c = 0; c < 3; c++) {
      double p[10] = {0}, q[10] = {0}, Mc[10];
      rel5_pmul(e[mi[c][0]], 4, rel5_qidx, e[mi[c][1]], p);
      rel5_pmul(e[mi[c][2]], 4, rel5_qidx, e[mi[c][3]], q);
      for (int m = 0; m < 10; m++) Mc[m] = p[m] - q[m];
      rel5_pmul(Mc, 10, rel5_cidx, e[c], D);
    }
    memcpy(A[9], D, sizeof(D));
  }
  /* 3. Gauss-Jordan on the left 10x10 block (A0 keeps the cubics for the polish) */
  double A0[10][20];
  memcpy(A0, A, sizeof(A));
  double amax = 0.0;
  for (int i = 0; i < 10; i++)
    for (int j = 0; j < 20; j++) amax = fabs(A[i][j]) > amax ? fabs(A[i][j]) : amax;
  const double tol = REL5_PIVOT_TOL * amax;
  for (int k = 0; k < 10; k++) {
    int p = k;
    for (int i = k + 1; i < 10; i++)
      if (fabs(A[i][k]) > fabs(A[p][k])) p = i;
    const double piv = A[p][k];
    if (!(fabs(piv) >= tol) || !(amax > 0.0)) return 0;
    for (int j = 0; j < 20; j++) { const double t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
    for (int j = 0; j < 20; j++) A[k][j] = A[k][j] / piv;
    for (int i = 0; i < 10; i++) {
      if (i == k) continue;
      const double f = A[i][k];
      for (int j = 0; j < 20; j++) A[i][j] = A[i][j] - f * A[k][j];
    }
  }
  /* B(z) (ascending powers, 5 each) and n(z) */
  double Bp[9][5], n[13] = {0};
  for (int r = 0; r < 3; r++) {
    const double *g = A[4 + 2 * r] + 10, *h = A[5 + 2 * r] + 10;
    for (int c = 0; c < 2; c++) {
      const int o = 3 * c;
      double* b = Bp[3 * r + c];
      b[0] = g[o + 2]; b[1] = g[o + 1] - h[o + 2]; b[2] = g[o] - h[o + 1]; b[3] = -h[o]; b[4] = 0.0;
    }
    double* b = Bp[3 * r + 2];
    b[0] = g[9]; b[1] = g[8] - h[9]; b[2] = g[7] - h[8]; b[3] = g[6] - h[7]; b[4] = -h[6];
  }
  {
    static const int mi[3][4] = {{4, 8, 5, 7}, {5, 6, 3, 8}, {3, 7, 4, 6}};
    for (int c = 0; c < 3; c++) {
      double p[9] = {0}, q[9] = {0}, Mc[9];
      rel5_upmul(Bp[mi[c][0]], 5, Bp[mi[c][1]], 5, p);
      rel5_upmul(Bp[mi[c][2]], 5, Bp[mi[c][3]], 5, q);
      for (int m = 0; m < 9; m++) Mc[m] = p[m] - q[m];
      rel5_upmul(Bp[c], 5, Mc, 9, n);
    }
  }
  /* real roots of n by the derivative cascade */
  double D[11][11];
  memcpy(D[10], n, 11 * sizeof(double));
  for (int d = 10; d >= 1; d--)
    for (int i = 0; i < d; i++) D[d - 1][i] = D[d][i + 1] * (double)(i + 1);
  double bmax = 0.0;
  for (int i = 0; i < 10; i++) {
    const double q = fabs(n[i] / n[10]);
    bmax = q > bmax ? q : bmax;
  }
  const double bnd = 1.0 + bmax;
  if (!(bnd < INFINITY)) return 0;
  double rt[10];
  int nr = 0;
  for (int d = 1; d <= 10; d++) {
    double nrt[10];
    int nn = 0;
    for (int k = 0; k <= nr; k++) {
      double z;
      if (rel5_root(D[d], d, D[d - 1], k == 0 ? -bnd : rt[k - 1], k == nr ? bnd : rt[k], &z)) nrt[nn++] = z;
    }
    memcpy(rt, nrt, sizeof(double) * (size_t)nn);
    nr = nn;
  }
  if (det) det->n_roots = nr;
  /* 4-5. per root: E, its four decompositions and their qualities */
  double best = INFINITY;
  int found = 0;
  for (int k = 0; k < nr; k++) {
    const double z = rt[k];
    double Bz[9], v[3], nv;
    for (int i = 0; i < 9; i++) Bz[i] = rel5_horner(Bp[i], 4, z);
    rel5_cross_max(Bz, Bz + 3, Bz + 6, v, &nv);
    double xyz[3] = {v[0] / v[2], v[1] / v[2], z};
    rel5_polish(A0, xyz);
    const double x = xyz[0], y = xyz[1];
    double E[9];
    for (int i = 0; i < 9; i++) E[i] = ((x * basis[0][i] + y * basis[1][i]) + xyz[2] * basis[2][i]) + basis[3][i];
    double fro = 0.0;
    for (int i = 0; i < 9; i++) fro = i == 0 ? E[i] * E[i] : fro + E[i] * E[i];
    const double sc = sqrt(0.5 * fro);
    for (int i = 0; i < 9; i++) E[i] = E[i] / sc;
    double col[3][3], b[3], nb, cof[9], bx[9];
    for (int j = 0; j < 3; j++)
      for (int i = 0; i < 3; i++) col[j][i] = E[3 * i + j];
    rel5_cross_max(col[0], col[1], col[2], b, &nb);
    const double bn = sqrt(nb);
    for (int i = 0; i < 3; i++) b[i] = b[i] / bn;
    cross3(E + 3, E + 6, cof); cross3(E + 6, E, cof + 3); cross3(E, E + 3, cof + 6);
    for (int j = 0; j < 3; j++) {
      double u[3];
      cross3(b, col[j], u);
      for (int i = 0; i < 3; i++) bx[3 * i + j] = u[i];
    }
    if (det) { det->z[k] = z; memcpy(det->E[k], E, sizeof(E)); }
    for (int c = 0; c < 4; c++) {
      double M[12], ti[3];
      for (int r = 0; r < 3; r++) {
        for (int j = 0; j < 3; j++) M[4 * r + j] = c < 2 ? cof[3 * r + j] - bx[3 * r + j] : cof[3 * r + j] + bx[3 * r + j];
        M[4 * r + 3] = c & 1 ? -b[r] : b[r];
      }
      for (int r = 0; r < 3; r++) ti[r] = -((M[r] * M[3] + M[4 + r] * M[7]) + M[8 + r] * M[11]);
      double q = 0.0;
      for (int i = 0; i < REL5_SAMPLE; i++) {
        const double *a = P->f1 + 3 * (size_t)s[i], *bb = P->f2 + 3 * (size_t)s[i];
        double X[3], r2[3], Xn[3], rn[3];
        rel5_triangulate(M, ti, a, bb, X, r2);
        const double n1 = sqrt((X[0] * X[0] + X[1] * X[1]) + X[2] * X[2]), n2 = sqrt((r2[0] * r2[0] + r2[1] * r2[1]) + r2[2] * r2[2]);
        for (int r = 0; r < 3; r++) { Xn[r] = X[r] / n1; rn[r] = r2[r] / n2; }
        const double term = (1.0 - dot3(a, Xn)) + (1.0 - dot3(bb, rn));
        q = i == 0 ? term : q + term;
      }
      if (det) { memcpy(det->cand[k][c], M, sizeof(M)); det->quality[k][c] = q; }
      if (isfinite(q) && q < best) {
        best = q; found = 1;
        memcpy(model, M, sizeof(M));
      }
    }
  }
  return found && finite_n(model, 12);
}

/* a camera: offset 0, rotation I */
static const double rel5_identity_cam[12] = {0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1};

/* inlier count (and flags, nullable) of model M over the problem: ransac_rel_oracle.c's rel_count with one identity camera per
 * side */
static int rel5_count(const rel5_problem* P, const double* M, double threshold, uint8_t* mask) {
  double q[15];
  pair_model(M, rel5_identity_cam, rel5_identity_cam + 3, rel5_identity_cam, rel5_identity_cam + 3, q);
  for (int r = 0; r < 3; r++) q[12 + r] = -((q[r] * q[3] + q[4 + r] * q[7]) + q[8 + r] * q[11]);
  int cnt = 0;
  for (int i = 0; i < P->n; i++) {
    const int in = rel_score(q, q + 12, P->f1 + 3 * (size_t)i, P->f2 + 3 * (size_t)i, P->s1[i], P->s2[i]) < threshold;
    if (mask) mask[i] = (uint8_t)in;
    cnt += in;
  }
  return cnt;
}

/* one problem's RANSAC over its samples [n_samples][5]: the selection of ora_ransac_noncentral_relative_pose with sample size 5;
 * outputs of this problem (g0: index of its first sample in the per-sample outputs) */
static void rel5_ransac_problem(const rel5_problem* P, const int32_t* samples, int n_samples, double threshold, int max_iterations,
                                double probability, int32_t* best_sample, double* best_model, int32_t* best_count, int32_t* iterations,
                                int32_t* consumed, uint8_t* inlier_mask, size_t g0, double* sample_model, uint8_t* sample_valid,
                                int32_t* sample_count) {
  const double log_p = log(1.0 - probability), eps = 2.220446049250313e-16;
  const long long max_skip = 10LL * max_iterations;
  const int n = P->n;
  int best = -1, best_n = 0, it = 0, s_used = 0;
  long long skipped = 0;
  double k = (double)max_iterations, bm[12] = {0};
  for (int s = 0; s < n_samples; s++) {
    const int running = it < max_iterations && (double)it < k && skipped < max_skip;
    if (!running && !sample_model) break;
    double M[12] = {0};
    const int valid = rel5_hypothesis(P, samples + REL5_SAMPLE * (size_t)s, M, NULL);
    if (!valid) memset(M, 0, sizeof(M));
    const int cnt = valid ? rel5_count(P, M, threshold, NULL) : 0;
    if (sample_model) {
      const size_t g = g0 + s;
      memcpy(sample_model + 12 * g, M, sizeof(M)); sample_valid[g] = (uint8_t)valid; sample_count[g] = cnt;
    }
    if (!running) continue;
    s_used++;
    if (!valid) { skipped++; continue; }
    if (cnt > best_n) {
      best_n = cnt; best = s; memcpy(bm, M, sizeof(bm));
      const double w = (double)cnt / (double)n;
      double wp = w;
      for (int e = 1; e < REL5_SAMPLE; e++) wp = wp * w;
      double pno = 1.0 - wp;
      pno = pno > eps ? pno : eps;
      pno = pno < 1.0 - eps ? pno : 1.0 - eps;
      k = log_p / log(pno);
    }
    it++;
  }
  *best_sample = best; *best_count = best_n; *iterations = it; *consumed = s_used;
  memcpy(best_model, bm, sizeof(bm));
  if (inlier_mask) {
    if (best >= 0) rel5_count(P, bm, threshold, inlier_mask);
    else memset(inlier_mask, 0, (size_t)n);
  }
}

/* one 5-point sample of a central problem (n correspondences): → model [12] (zeros if invalid); n_roots, z [10] (ascending),
 * E [10][9] (scaled), cand [10][4][12], quality [10][4] (all nullable together) for the real roots; returns valid */
API int ora_rel5(int n, const double* f1, const double* f2, const int32_t* sample, double* model, int32_t* n_roots, double* z, double* E,
                 double* cand, double* quality) {
  const rel5_problem P = {n, f1, f2, NULL, NULL};
  rel5_detail d;
  memset(&d, 0, sizeof(d));
  memset(model, 0, 96);
  const int v = rel5_hypothesis(&P, sample, model, &d);
  if (!v) memset(model, 0, 96);
  if (n_roots) {
    *n_roots = d.n_roots;
    memcpy(z, d.z, sizeof(d.z)); memcpy(E, d.E, sizeof(d.E)); memcpy(cand, d.cand, sizeof(d.cand)); memcpy(quality, d.quality, sizeof(d.quality));
  }
  return v;
}

/* Same arguments and outputs as cvb_ransac_central_relative_pose_batch (flattened), the selection with sample size 5. */
API void ora_ransac_central_relative_pose(int n_prob, const int32_t* prob_ptr, const double* f1, const double* f2, const double* sigma1,
                                          const double* sigma2, const int32_t* samples, int n_samples, double threshold, int max_iterations,
                                          double probability, int32_t* best_sample, double* best_model, int32_t* best_count,
                                          int32_t* iterations, int32_t* consumed, uint8_t* inlier_mask, double* sample_model,
                                          uint8_t* sample_valid, int32_t* sample_count) {
#pragma omp parallel for schedule(dynamic, 1)
  for (int pi = 0; pi < n_prob; pi++) {
    const int off = prob_ptr[pi], n = prob_ptr[pi + 1] - prob_ptr[pi];
    const rel5_problem P = {n, f1 + 3 * (size_t)off, f2 + 3 * (size_t)off, sigma1 + off, sigma2 + off};
    rel5_ransac_problem(&P, samples + REL5_SAMPLE * (size_t)pi * n_samples, n_samples, threshold, max_iterations, probability,
                        best_sample + pi, best_model + 12 * (size_t)pi, best_count + pi, iterations + pi, consumed + pi,
                       inlier_mask ? inlier_mask + off : NULL, (size_t)pi * n_samples, sample_model, sample_valid, sample_count);
  }
}
