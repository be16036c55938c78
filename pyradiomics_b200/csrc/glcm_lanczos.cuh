// MCC eigen-tasks of large level graphs (13..18 nodes; only the three axis angles have enough pairs for
// that): second largest |eigenvalue| of M = D^-1/2 A D^-1/2, A = co-occurrence counts of ONE angle whose
// level graph is connected and not bipartite (phase A filters those), D = diag(row sums R).
//   * the window is loaded PERMUTED so that the angle axis is the fastest window coordinate: the 18 pairs
//     are the static position pairs (p, p+1), p % 3 < 2 -- no per-slot tables, all pair code is unrolled;
//   * level classes are 27-bit position masks (__vcmpeq4 on the packed window), node i = i-th class in
//     order of its lowest position, so R_i and everything per node sits in registers with STATIC indices;
//   * the recurrence runs in "random-walk" coordinates y = D^-1/2 q with the D-inner product: the operator
//     is W = D^-1 A, i.e. (W y)_i = (sum of y over the neighbour endpoints of i) / R_i -- no edge weights,
//     the known top eigenvector is the constant vector, and deflating it is a scalar shift;
//   * the Lanczos vectors y0, y1 and R live in registers (fp64, no float storage, no start-vector
//     heuristics beyond a fixed generic start); the only dynamically indexed data are two per-thread
//     shared-memory vectors U (= y1) and S (neighbour sums), laid out [node][thread] so a warp's 64-bit
//     accesses are always two conflict-free wavefronts whatever the node indices are;
//   * every loop has a compile-time trip count (N = 14 / 16 / 18 by size class): a warp's lanes never
//     diverge; a breakdown (invariant subspace) just continues with zero vectors, which leaves decoupled
//     zero eigenvalues in the tridiagonal -- harmless for max(|hi|, |lo|).  Padded nodes (n < N) contribute exact zeros
//     to every sum, and the eigenvalue search runs over the template's whole (N-1) x (N-1) tridiagonal.  A task's size
//     class fixes its template, so its bits are reproducible; results from different templates agree to rounding, not
//     to the bit.
// __host__ __device__: tests/host_emul checks the arithmetic against LAPACK on the CPU box (test-only).
#pragma once
// (included from the middle of glcm_fast.cuh: needs GlcmSolveTables, glcm_eq_positions, tridiag_extreme_pair_static)

namespace rb {

constexpr uint32_t LZ_LOW = 0x36DB6DBu;       // window positions p (a*9 + b*3 + c) with c < 2: lower ends of the pairs (p, p+1)
constexpr int LZ_ACC = 3;                     // interleaved partial sums per reduction
constexpr int LZ_NARR = 5;                    // per-thread shared arrays: U, S, IR, D, E (N doubles each)
constexpr double GF_BREAKDOWN = 1e-10;        // Lanczos breakdown: residual norms at or below this continue with zeros

RB_HD constexpr int lz_smem_doubles(int N) { return LZ_NARR * N; }

// wl: the 27 window levels with the angle axis as the FASTEST coordinate (0 = unmasked / outside);
// sm: per-thread scratch of LZ_NARR*N doubles with element stride st.
// Returns the second largest |eigenvalue|; *n_out = number of level nodes (> N: nothing computed, NaN).
template <int N, class TT>
RB_HD double glcm_lanczos_axis(const int* wl, const TT& T, double* sm, int st, int* n_out, bool live = true) {
  double* const U = sm;
  double* const S = sm + (size_t)N * st;
  double* const IR = sm + (size_t)2 * N * st;
  double* const D = sm + (size_t)3 * N * st;
  double* const E = sm + (size_t)4 * N * st;
  uint32_t W7[7];
#pragma unroll
  for (int k = 0; k < 7; k++) {
    uint32_t v = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) if (4 * k + b < 27) v |= (uint32_t)wl[4 * k + b] << (8 * b);
    W7[k] = v;
  }
  const uint32_t NZ = ~glcm_eq_positions(W7, 0u) & 0x7FFFFFFu;
  const uint32_t VL = NZ & (NZ >> 1) & LZ_LOW;             // valid pairs, by their lower position
  const uint32_t VH = VL << 1;
  uint32_t Urem = VL | VH;                                 // endpoint positions not yet assigned to a class
  // ---- level classes in order of their lowest position; R_i = endpoint multiplicity (row sum of A)
  double Rd[N];
  uint32_t plane[5] = {0, 0, 0, 0, 0};                     // bit p of plane[b] = bit b of the node index of position p
  int n = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t Ec = 0;
    if (Urem) {
      const int p = RB_CTZ(Urem);
      const uint32_t lev = (W7[p >> 2] >> (8 * (p & 3))) & 255u;
      Ec = glcm_eq_positions(W7, lev);
      Urem &= ~Ec;
      n++;
    }
    const int Ri = RB_POPC(Ec & VL) + RB_POPC(Ec & VH);
    Rd[i] = (double)Ri;
    IR[(size_t)i * st] = T.rinv[Ri];
#pragma unroll
    for (int b = 0; b < 5; b++) if (i >> b & 1) plane[b] |= Ec;
  }
  *n_out = n + (Urem ? RB_POPC(Urem) : 0);                 // (> N when classes are left over)
  if (Urem) return NAN;
  // node index of both ends of the 18 static pairs, 5 bits each
  uint32_t ida[3] = {0, 0, 0}, idb[3] = {0, 0, 0};          // 6 pairs per word
#pragma unroll
  for (int t = 0; t < 18; t++) {
    const int p = (t / 2) * 3 + (t % 2);                   // lower position of pair t
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int k = 0; k < 5; k++) { a |= ((plane[k] >> p) & 1u) << k; b |= ((plane[k] >> (p + 1)) & 1u) << k; }
    ida[t / 6] |= a << (5 * (t % 6));
    idb[t / 6] |= b << (5 * (t % 6));
  }
  // ---- start vector (generic fixed components), D-orthogonal to the constant vector, D-normalised
  double y0[N], y1[N];
  double Ssum = 0, dot = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    y1[i] = Rd[i] != 0.0 ? T.lz0[i] : 0.0;
    y0[i] = 0.0;
    Ssum += Rd[i];
    dot += Rd[i] * y1[i];
  }
  const double cc = 1.0 / Ssum;                            // <1,1>_D = S: the top eigenvector is 1/sqrt(S)
  double nrm = 0;
  {
    const double sh = dot * cc;
#pragma unroll
    for (int i = 0; i < N; i++) { y1[i] = Rd[i] != 0.0 ? y1[i] - sh : 0.0; nrm += Rd[i] * y1[i] * y1[i]; }
  }
  {
    const double inrm = 1.0 / sqrt(nrm);
#pragma unroll
    for (int i = 0; i < N; i++) y1[i] *= inrm;
  }
  double beta = 0;
  E[0] = 0;
  // ---- N-1 Lanczos steps (the deflated space has n-1 <= N-1 dimensions; see the file header for breakdowns)
  for (int j = 0; j < N - 1; j++) {
#pragma unroll
    for (int i = 0; i < N; i++) { U[(size_t)i * st] = y1[i]; S[(size_t)i * st] = 0.0; }
    // neighbour sums: S[a] += y[b], S[b] += y[a] for every valid pair (a self pair adds 2 y[a])
#pragma unroll
    for (int t = 0; t < 18; t++) {
      const int p = (t / 2) * 3 + (t % 2);
      if (VL >> p & 1u) {
        const size_t a = (size_t)((ida[t / 6] >> (5 * (t % 6))) & 31u) * st, b = (size_t)((idb[t / 6] >> (5 * (t % 6))) & 31u) * st;
        const double ua = U[a], ub = U[b];
        S[a] += ub;
        S[b] += ua;
      }
    }
    // z = W y1 - beta y0 (kept in y0's registers); alpha = <y1, W y1>_D = sum y1_i s_i.  Every reduction below runs
    // on LZ_ACC interleaved partial sums: with two warps per scheduler a single 18-long DFMA chain is exposed latency.
    double al[LZ_ACC];
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) al[k] = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
      const double s = S[(size_t)i * st];
      al[i % LZ_ACC] += y1[i] * s;
      y0[i] = s * IR[(size_t)i * st] - beta * y0[i];
    }
    double alpha = 0;
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) alpha += al[k];
    // z -= alpha y1; then re-orthogonalise against the deflated constant vector and y1
    double dvp[LZ_ACC], c1p[LZ_ACC];
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) { dvp[k] = 0; c1p[k] = 0; }
#pragma unroll
    for (int i = 0; i < N; i++) {
      y0[i] -= alpha * y1[i];
      const double g = Rd[i] * y0[i];
      dvp[i % LZ_ACC] += g; c1p[i % LZ_ACC] += g * y1[i];
    }
    double dv = 0, c1 = 0;
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) { dv += dvp[k]; c1 += c1p[k]; }
    dv *= cc;                                              // <z, 1>_D / <1,1>_D
    double nbp[LZ_ACC];
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) nbp[k] = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
      const double zi = Rd[i] != 0.0 ? y0[i] - dv - c1 * y1[i] : 0.0;
      y0[i] = zi;
      nbp[i % LZ_ACC] += Rd[i] * zi * zi;
    }
    double nb = 0;
#pragma unroll
    for (int k = 0; k < LZ_ACC; k++) nb += nbp[k];
    D[(size_t)j * st] = alpha;
    nb = sqrt(nb);
    const bool ok = nb > GF_BREAKDOWN;
    const double inb = ok ? 1.0 / nb : 0.0;
    beta = ok ? nb : 0.0;
    if (j + 1 < N - 1) E[(size_t)(j + 1) * st] = beta;
    // rotate: new y1 = z / nb, new y0 = old y1
#pragma unroll
    for (int i = 0; i < N; i++) { const double t1 = y1[i]; y1[i] = y0[i] * inb; y0[i] = t1; }
  }
  // both extreme eigenvalues of the (N-1) x (N-1) tridiagonal, held in the registers the vectors have freed
  double d[N - 1], e[N - 1];
#pragma unroll
  for (int i = 0; i < N - 1; i++) { d[i] = D[(size_t)i * st]; e[i] = E[(size_t)i * st]; }
  double hi, lo;
  // padded / broken-down rows are decoupled zero eigenvalues, harmless for max(|hi|,|lo|)
  tridiag_extreme_pair_static<N - 1, false>(d, e, &hi, &lo, live && n >= 2);
  return fmax(fabs(hi), fabs(lo));
}

// eigen-task entry: w = the voxel's 27 window levels in natural (z,y,x) order, s = angle slot 0 / 1 / 2 = the z / y / x
// axis angle (glcm_fast_build_tables puts the three axis angles first).  Permutes the window so that the angle axis is
// the fastest coordinate and runs the solver.
template <int N, class TT>
RB_HD double glcm_lanczos_task(const uint8_t* w, int ws, const TT& T, int s, double* sm, int st, int* n_out, bool live = true) {
  int wl[27];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++)
#pragma unroll
      for (int c = 0; c < 3; c++) {
        // slot 2 (x): (z,y,x) = (a,b,c); slot 1 (y): (a,c,b); slot 0 (z): (c,a,b)
        const int v2 = w[(a * 9 + b * 3 + c) * ws], v1 = w[(a * 9 + c * 3 + b) * ws], v0 = w[(c * 9 + a * 3 + b) * ws];
        wl[a * 9 + b * 3 + c] = s == 2 ? v2 : s == 1 ? v1 : v0;
      }
  return glcm_lanczos_axis<N>(wl, T, sm, st, n_out, live);
}

// Level graph of one angle in POSITION space: eq[p*es] = mask of the window positions holding the level of position p
// (a class), EA = lower ends of the valid pairs, every pair is (p, p + dsh), U = all pair ends.  One breadth-first
// sweep over class masks answers both questions of the MCC classification: is the graph connected, and is it
// bipartite (2-colourable; `selfpair` = some level is paired with itself, which rules that out and lets the sweep
// run with one colour).  A class joins each colour at most once, so the closure loops run <= 2 nlev times in total.
RB_HD void glcm_graph_scan(const uint32_t* eq, int es, uint32_t EA, int dsh, uint32_t U, bool selfpair, bool* connected,
                           bool* bipartite, bool stop_at_odd_cycle = false) {
  const int p0 = RB_CTZ(EA);
  if (selfpair) {
    uint32_t Cm = eq[(size_t)p0 * es], F = Cm;
    while (F) {
      uint32_t Pn = (((F & EA) << dsh) | ((F >> dsh) & EA)) & ~Cm;     // partner positions not reached yet
      F = 0;
      while (Pn) { const uint32_t c = eq[(size_t)RB_CTZ(Pn) * es]; F |= c; Pn &= ~c; }
      Cm |= F;
    }
    *connected = (U & ~Cm) == 0;
    *bipartite = false;
    return;
  }
  uint32_t CA = eq[(size_t)p0 * es], CB = 0, FA = CA, FB = 0;
  while (FA | FB) {
    uint32_t PA = (((FA & EA) << dsh) | ((FA >> dsh) & EA)) & ~CB;     // partners of the new A positions: must be B
    uint32_t PB = (((FB & EA) << dsh) | ((FB >> dsh) & EA)) & ~CA;
    FA = 0; FB = 0;
    while (PA) { const uint32_t c = eq[(size_t)RB_CTZ(PA) * es]; FB |= c; PA &= ~c; }
    while (PB) { const uint32_t c = eq[(size_t)RB_CTZ(PB) * es]; FA |= c; PB &= ~c; }
    CA |= FA; CB |= FB;
    if (stop_at_odd_cycle && (CA & CB)) break;   // the caller only wants the colouring: an odd cycle settles it
  }
  *connected = (U & ~(CA | CB)) == 0;           // (not meaningful after an early stop)
  *bipartite = (CA & CB) == 0;                   // a class that needs both colours closes an odd cycle
}

}  // namespace rb
