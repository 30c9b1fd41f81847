// Newton Hessian  H = M + J^T D_active J  and its Cholesky solve, exploiting the block structure of the scene.
//
// The mass matrix is block diagonal over kinematic trees (the arm + one block per object).  A contact couples two trees
// only when both of its bodies are dynamic and belong to different trees.  Trees that no such contact (or equality row)
// touches are "uncoupled": their Hessian block is assembled, factorised and solved by an 8-lane group each, several trees at a
// time.  Coupled trees (e.g. arm + grasped object, touching objects of a pile) form connected components ("islands"); the Hessian
// is block diagonal over islands and each island is factorised as ONE dense matrix by one warp.
//
// Storage (r02): nothing is kept at global dof indices any more.  The region L.H (nv (nv + 1) / 2 doubles, the size of the full
// packed triangle, which is an upper bound of what follows) is handed out per Hessian build: one packed lower-triangular BLOCK per
// uncoupled tree (n_t (n_t + 1) / 2) and one per island (n_isl (n_isl + 1) / 2, island-local row order = ascending dof order),
// back to back.  Entry (i, j) of a block lives at  off + r (r + 1) / 2 + c  with r, c the block-local indices, so the factorisation
// loops run over dense local indices (the r01 version indexed the global triangle through a dof list: 247 KB of scattered entries
// per environment in the 40-object scene, ~12 integer instructions per multiply-add).  Included by ge_solver.cuh.
#pragma once

#define HIDX(i, j) (((i) * ((i) + 1)) / 2 + (j))
#define GE_TLIST 16  // row length of the per-tree int list: GE_TCAP contact ids + the tree's block offset in the last slot
#define GE_TCAP (GE_TLIST - 1)  // contacts per uncoupled tree handled by the group path (more -> the tree takes the coupled path)
#define GE_GROUP 8  // lanes per kinematic tree in the uncoupled-tree path (trees with more dofs use the coupled path)

namespace ge {

__device__ __forceinline__ int tree_of_body(int b) {
  int d = c_m.body_lastdof[b];
  return d < 0 ? -1 : c_m.dof_treeindex[d];
}

// active-set weights applied to one Jacobian column: t = W J  (W00 = D nact, W0k = D mu_k (a+ - a-), Wkk = D mu_k^2 (a+ + a-))
__device__ __forceinline__ void weight_column(const double* c, int dim, int mask, const double* J, double* t) {
  double D = c[C_D];
  if (dim == 1) { t[0] = D * J[0]; return; }
  int nact = __popc(mask);
  double t0 = nact * J[0];
  for (int k = 1; k < dim; k++) {
    int ap = (mask >> (2 * (k - 1))) & 1, an = (mask >> (2 * (k - 1) + 1)) & 1;
    double mu = c[C_MU + k - 1];
    t0 += mu * (ap - an) * J[k];
    t[k] = D * mu * ((ap - an) * J[0] + mu * (ap + an) * J[k]);
  }
  t[0] = D * t0;
}
__device__ __forceinline__ void jac_column(const double* c, int dim, const double* cd, double sgn, double* J) {
  double pu[3];
  for (int k = 0; k < dim; k++) {
    if (k < 3) { v3cross(pu, c + C_POS, c + C_FRAME + 3 * k); J[k] = sgn * (v3dot(c + C_FRAME + 3 * k, cd + 3) + v3dot(pu, cd)); }
    else J[k] = sgn * v3dot(c + C_FRAME + 3 * (k - 3), cd);
  }
}

// owner warp of the island a coupled tree belongs to (CTA-per-env build: islands are dealt out to the warps; their Hessian blocks
// are disjoint, so the warps never touch the same entry)
// The owner is chosen per Hessian build by longest-processing-time-first over the islands' cubic cost (build_hessian) and kept in slot 1
// of the representative's list row: with `island % GE_NW` one warp regularly held the two largest islands of a pile while the others
// idled at the next barrier.
__device__ __forceinline__ int island_owner(const int* island, const int* tlist, int t) { return tlist[island[t] * 16 + 1]; }
// per-tree bookkeeping of one Hessian build: block offset (of the tree's own block, or of its island's block) and, for coupled trees,
// the tree's first row inside the island block
#define T_HOFF(tlist, t) (tlist)[(t) * GE_TLIST + GE_TCAP]

__device__ __noinline__ void build_hessian(double* ws, int* wi, int ncon, int nsr, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  double* H = ws + L.H;  // (CTA-per-env build: re-pointed at the env's HBM overflow row below if this build's blocks exceed L.hcap)
  const double *qM = ws + L.qM, *cdof = ws + L.cdof;
  const int wl = lane & 31, wid = lane >> 5;
  int* tcoupled = wi + L.i_tcoupled;
  int *tcount = wi + L.i_tcount, *tlist = wi + L.i_tlist, *island = wi + L.i_island;  // tcount: #contacts (uncoupled) / first island row (coupled)
  // ---- which trees are coupled to another tree by an active constraint (trees wider than a lane group take the coupled path too)
  LANE_LOOP(t, m.ntree) { tcoupled[t] = m.tree_dofnum[t] > GE_GROUP ? 1 : 0; island[t] = t; }
  gsync();
  LANE_LOOP(ci, ncon) {
    if (!wi[L.i_cact + ci]) continue;
    int t1 = wi[L.i_ct1 + ci], t2 = wi[L.i_ct2 + ci];
    if (t1 >= 0 && t2 >= 0 && t1 != t2) { tcoupled[t1] = 1; tcoupled[t2] = 1; }
  }
  LANE_LOOP(i, nsr) {
    if (!wi[L.i_sract + i]) continue;
    int A = wi[L.i_srA + i], B = wi[L.i_srB + i];
    if (B >= 0 && m.dof_treeindex[A] != m.dof_treeindex[B]) { tcoupled[m.dof_treeindex[A]] = 1; tcoupled[m.dof_treeindex[B]] = 1; }
  }
  gsync();
  // ---- per-tree lists of the active contacts that live entirely inside one uncoupled tree (one lane per tree scans the contacts)
  LANE_LOOP(t, m.ntree) {
    int cnt = 0;
    if (!tcoupled[t]) {
      for (int ci = 0; ci < ncon; ci++)
        if (wi[L.i_cact + ci] && (wi[L.i_ct1 + ci] == t || wi[L.i_ct2 + ci] == t)) { if (cnt < GE_TCAP) tlist[t * GE_TLIST + cnt] = ci; cnt++; }
      if (cnt > GE_TCAP) { tcoupled[t] = 1; cnt = 0; }  // too many contacts for the list: this tree takes the coupled path
    }
    tcount[t] = cnt;
  }
  gsync();
  bool any_coupled = false;
  for (int t = 0; t < m.ntree; t++) any_coupled |= tcoupled[t] != 0;
  // ---- islands of the coupled trees.  Label propagation: every tree starts with its own index, edges pull both ends to the smaller
  // label until nothing changes (the fixed point - the smallest tree index of the component - does not depend on the update order).
  if (any_coupled) {
    for (int iter = 0; iter < m.ntree; iter++) {
      bool changed = false;
      LANE_LOOP(ci, ncon) {
        if (!wi[L.i_cact + ci]) continue;
        int t1 = wi[L.i_ct1 + ci], t2 = wi[L.i_ct2 + ci];
        if (t1 < 0 || t2 < 0 || t1 == t2) continue;
        int a = ((volatile int*)island)[t1], b = ((volatile int*)island)[t2];
        if (a != b) { int mn = a < b ? a : b; atomicMin(island + t1, mn); atomicMin(island + t2, mn); changed = true; }
      }
      LANE_LOOP(i, nsr) {
        if (!wi[L.i_sract + i]) continue;
        int A = wi[L.i_srA + i], B = wi[L.i_srB + i];
        if (B < 0) continue;
        int t1 = m.dof_treeindex[A], t2 = m.dof_treeindex[B];
        if (t1 == t2) continue;
        int a = ((volatile int*)island)[t1], b = ((volatile int*)island)[t2];
        if (a != b) { int mn = a < b ? a : b; atomicMin(island + t1, mn); atomicMin(island + t2, mn); changed = true; }
      }
      changed = group_any(changed);
      gsync();
      if (!changed) break;
    }
    // The labels were merged with atomicMin, which is resolved in L2 and leaves any copy of the line in this SM's L1 as it was; the plain
    // loads below (and in cholesky_solve) could then see pre-merge labels - and, in the CTA-per-env build, DIFFERENT warps different ones
    // depending on when the line is evicted (r02d: garbage Hessian blocks -> non-finite states under load; gone with -Xptxas -dlcm=cg).
    // Read the final labels past L1 once and write them back with ordinary stores, which L1 does track.
    {
      const int ta = lane, tb = lane + GE_LANES;  // (ntree <= 2 * GE_LANES is checked at ge_create)
      const int la = ta < m.ntree ? ((volatile int*)island)[ta] : 0, lb = tb < m.ntree ? ((volatile int*)island)[tb] : 0;
      gsync();
      if (ta < m.ntree) island[ta] = la;
      if (tb < m.ntree) island[tb] = lb;
      gsync();
    }
    // first row of every coupled tree inside its island block (members in ascending tree order); the representative also records the
    // island's size (first slot of its - otherwise unused - contact list row)
    LANE_LOOP(t, m.ntree) {
      if (!tcoupled[t]) continue;
      int isl = island[t], r0 = 0;
      for (int tt = isl; tt < t; tt++) if (tcoupled[tt] && island[tt] == isl) r0 += m.tree_dofnum[tt];
      tcount[t] = r0;
      if (isl == t) { int n = 0; for (int v = t; v < m.ntree; v++) if (tcoupled[v] && island[v] == t) n += m.tree_dofnum[v]; tlist[t * GE_TLIST] = n; }
    }
    gsync();
  }
  // ---- block offsets: trees in ascending order, an uncoupled tree takes its own block, an island takes its block at its representative
  LANE_LOOP(t, m.ntree) {
    int off = 0;
    const int stop = tcoupled[t] ? island[t] : t;
    for (int u = 0; u < stop; u++) {
      int n;
      if (!tcoupled[u]) n = m.tree_dofnum[u];
      else if (island[u] == u) n = tlist[u * GE_TLIST];
      else continue;
      off += n * (n + 1) / 2;
    }
    T_HOFF(tlist, t) = off;
  }
#if GE_NW > 1
  {  // total size of this build's blocks (every thread adds up the same list)
    int tot = 0;
    for (int u = 0; u < m.ntree; u++) {
      int n;
      if (!tcoupled[u]) n = m.tree_dofnum[u];
      else if (island[u] == u) n = tlist[u * GE_TLIST];
      else continue;
      tot += n * (n + 1) / 2;
    }
    const bool ovf = tot > L.hcap;
    if (ovf) H = g_hovf;
    if (lane == 0) {
      wi[L.i_hflag] = ovf ? 1 : 0;
      // island -> warp: islands in descending order of size would be ideal; taking them in index order and always feeding the least
      // loaded warp is within a small factor and needs no sort
      long long load[GE_NW];
      for (int w = 0; w < GE_NW; w++) load[w] = 0;
      for (int u = 0; u < m.ntree; u++) {
        if (!tcoupled[u] || island[u] != u) continue;
        const long long n = tlist[u * GE_TLIST];
        int best = 0;
        for (int w = 1; w < GE_NW; w++) if (load[w] < load[best]) best = w;
        load[best] += n * n * n + 64 * n * n;
        tlist[u * GE_TLIST + 1] = best;
      }
    }
  }
#endif
  gsync();
  // ---- rows of M: zero fill of the whole block row, then the tree-sparse row of qM
  LANE_LOOP(i, m.nv) {
    const int t = m.dof_treeindex[i], lo = m.tree_dofadr[t];
    const int r0 = tcoupled[t] ? tcount[t] : 0, r = r0 + i - lo;
    double* row = H + T_HOFF(tlist, t) + r * (r + 1) / 2;
    for (int j = 0; j <= r; j++) row[j] = 0;
    int a = m.dof_Madr[i], k = 0;
    for (int j = i; j >= 0; j = m.dof_parentid[j], k++) row[r0 + j - lo] = qM[a + k];
  }
  gsync();
  // ---- uncoupled trees: one 8-lane group per tree, GE_LANES / 8 trees at a time, every group walking ITS OWN contact list so that
  // the groups really run concurrently (same instruction stream, different contacts).  Lane l of a group owns dof lo + l; the
  // contact's Jacobian block is rebuilt in registers and J^T W J is added to the tree's dense block through shuffles.
  {
    const int g = lane / GE_GROUP, l = lane % GE_GROUP, gw = wl & ~(GE_GROUP - 1);  // gw: first lane of my group inside my warp
    for (int t0 = 0; t0 < m.ntree; t0 += GE_LANES / GE_GROUP) {
      const int t = t0 + g;
      const bool valid = t < m.ntree && !tcoupled[t];
      const int lo = valid ? m.tree_dofadr[t] : 0, nt = valid ? m.tree_dofnum[t] : 0, cnt = valid ? tcount[t] : 0;
      double* Hb = H + (valid ? T_HOFF(tlist, t) : 0);
      const int mydof = lo + l;
      int maxcnt = cnt;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) maxcnt = max(maxcnt, __shfl_xor_sync(FULL, maxcnt, o));
      for (int n = 0; n < maxcnt; n++) {
        const bool act = n < cnt && l < nt;
        double J[6] = {0, 0, 0, 0, 0, 0}, tw[6] = {0, 0, 0, 0, 0, 0};
        if (act) {
          const int ci = tlist[t * GE_TLIST + n];
          const double* c = ws + L.con + ci * L.cstride;
          const int dim = wi[L.i_cdim + ci], t1 = wi[L.i_ct1 + ci], t2 = wi[L.i_ct2 + ci];
          // sign of my dof in the contact's dof list (chains of both bodies minus their common ancestors) from the per-body
          // bit masks over the tree-local dof index
          unsigned m1 = t1 == t ? (unsigned)m.body_chainmask[wi[L.i_cb1 + ci]] : 0u, m2 = t2 == t ? (unsigned)m.body_chainmask[wi[L.i_cb2 + ci]] : 0u;
          double sgn = ((m2 & ~m1) >> l & 1u) ? 1.0 : (((m1 & ~m2) >> l & 1u) ? -1.0 : 0.0);
          if (sgn != 0) { jac_column(c, dim, cdof + 6 * mydof, sgn, J); weight_column(c, dim, wi[L.i_cact + ci], J, tw); }
        }
        for (int f = 0; f < GE_GROUP; f++) {
          double h = 0;
          for (int k = 0; k < m.maxdim; k++) h += tw[k] * __shfl_sync(FULL, J[k], gw + f);
          if (act && l >= f && f < nt && h != 0.0) Hb[HIDX(l, f)] += h;
        }
      }
      __syncwarp();
      if (valid && l == 0)
        for (int i = 0; i < nsr; i++) {
          if (!wi[L.i_sract + i]) continue;
          int A = wi[L.i_srA + i], B = wi[L.i_srB + i];
          if (m.dof_treeindex[A] != t) continue;
          double D = srv(ws, SR_D, i), ca = srv(ws, SR_CA, i), cb = srv(ws, SR_CB, i);
          Hb[HIDX(A - lo, A - lo)] += D * ca * ca;
          if (B >= 0) {
            Hb[HIDX(B - lo, B - lo)] += D * cb * cb;
            int hi = A > B ? A : B, lw = A > B ? B : A;
            Hb[HIDX(hi - lo, lw - lo)] += D * ca * cb;
          }
        }
      __syncwarp();
    }
  }
  gsync();
  if (!any_coupled) return;
  // ---- coupled trees: warp-cooperative accumulation, one lane per dof of the contact; a contact belongs to the warp that owns its
  // island.  Block-local row of dof d of tree t: tcount[t] + d - tree_dofadr[t].
  for (int ci = 0; ci < ncon; ci++) {
    int mask = wi[L.i_cact + ci];
    if (!mask) continue;
    int b1 = wi[L.i_cb1 + ci], b2 = wi[L.i_cb2 + ci], t1 = wi[L.i_ct1 + ci], t2 = wi[L.i_ct2 + ci];
    const bool c1 = t1 >= 0 && tcoupled[t1], c2 = t2 >= 0 && tcoupled[t2];
    if (!(c1 || c2)) continue;
    const int tk = c1 ? t1 : t2;
    if (GE_NW > 1 && island_owner(island, tlist, tk) != wid) continue;
    double* Hb = H + T_HOFF(tlist, tk);
    const double* c = ws + L.con + ci * L.cstride;
    int dim = wi[L.i_cdim + ci];
    int i1 = m.body_lastdof[b1], i2 = m.body_lastdof[b2], n = 0, mydof = -1;
    double mysgn = 0;
    while (i1 != i2) {
      int e; double s;
      if (i2 > i1) { e = i2; s = 1.0; i2 = m.dof_parentid[i2]; } else { e = i1; s = -1.0; i1 = m.dof_parentid[i1]; }
      if (n == wl) { mydof = e; mysgn = s; }
      n++;
    }
    // The contact touches n dofs (12 for two free bodies), a warp has 32 lanes: P = 32 / n lanes share one row of the n x n update, lane
    // (r, p) takes the columns p, p + P, ...  Every entry still receives exactly one addition per contact, computed in the same order, so
    // the result does not depend on P.
    const int P = n > 0 && n <= 16 ? 32 / n : 1, r_ = n > 0 ? wl % n : 0, p_ = n > 0 ? wl / n : 0;
    const bool act = n > 0 && p_ < P && r_ < n;
    mydof = __shfl_sync(FULL, mydof, r_);
    mysgn = __shfl_sync(FULL, mysgn, r_);
    double J[6] = {0, 0, 0, 0, 0, 0}, t[6] = {0, 0, 0, 0, 0, 0};
    int myrow = -1;
    if (act) {
      jac_column(c, dim, cdof + 6 * mydof, mysgn, J);
      weight_column(c, dim, mask, J, t);
      const int tt = m.dof_treeindex[mydof];
      myrow = tcount[tt] + mydof - m.tree_dofadr[tt];
    }
    for (int j0 = 0; j0 < n; j0 += P) {
      const int j = j0 + p_;
      const bool v = act && j < n;
      const int src = v ? j : 0;  // lane j (p = 0) holds row j
      int rj = __shfl_sync(FULL, myrow, src);
      double h = 0;
      for (int k = 0; k < dim; k++) h += t[k] * __shfl_sync(FULL, J[k], src);
      if (v && myrow >= rj) Hb[HIDX(myrow, rj)] += h;
    }
    __syncwarp();
  }
  if (wl == 0)
    for (int i = 0; i < nsr; i++) {
      if (!wi[L.i_sract + i]) continue;
      int A = wi[L.i_srA + i], B = wi[L.i_srB + i];
      const int tA = m.dof_treeindex[A];
      if (!tcoupled[tA]) continue;
      if (GE_NW > 1 && island_owner(island, tlist, tA) != wid) continue;
      double* Hb = H + T_HOFF(tlist, tA);
      double D = srv(ws, SR_D, i), ca = srv(ws, SR_CA, i), cb = srv(ws, SR_CB, i);
      const int ra = tcount[tA] + A - m.tree_dofadr[tA];
      Hb[HIDX(ra, ra)] += D * ca * ca;
      if (B >= 0) {
        const int tB = m.dof_treeindex[B], rb = tcount[tB] + B - m.tree_dofadr[tB];
        Hb[HIDX(rb, rb)] += D * cb * cb;
        int hi = ra > rb ? ra : rb, lo = ra > rb ? rb : ra;
        Hb[HIDX(hi, lo)] += D * ca * cb;
      }
    }
  gsync();
}

// Dense Cholesky + forward/backward substitution of one tree block (packed lower triangle `Hb` of nt <= GE_GROUP rows, dofs lo ..
// lo + nt - 1) inside an 8-lane group, entirely in REGISTERS: lane l loads row l of the block once (static register indices, the loops
// are fully unrolled), the factorisation exchanges pivots / column entries through shuffles, nothing is written back to the matrix
// (the factor is used exactly once).  Rows l >= nt are padded with the identity.  x[lo + l] := sign * (H_block^-1 g)[l].
// (A shared-memory version spends most of its instructions in packed-index arithmetic, LDS/STS and three __syncwarp per column.)
__device__ __noinline__ void group_chol_solve(const double* Hb, int lo, int nt, int l, unsigned gmask, const double* g_, double* x, double sign) {
  const int row = lo + l;
  const bool mine = l < nt;
  double r[GE_GROUP], inv[GE_GROUP];
#pragma unroll
  for (int j = 0; j < GE_GROUP; j++) r[j] = (mine && j <= l) ? Hb[HIDX(l, j)] : (j == l ? 1.0 : 0.0);
  // right-looking Cholesky: after step j, r[j] holds L[l][j] (rows l > j), later columns carry the Schur complement.  Only 1 / L[j][j]
  // is ever needed (scaling of column j, the two substitutions), so the pivot is one reciprocal square root (rsqrt: <= 1 ulp).
#pragma unroll
  for (int j = 0; j < GE_GROUP; j++) {
    double d = __shfl_sync(gmask, r[j], j, GE_GROUP);
    if (d < GE_MINVAL) d = GE_MINVAL;
    inv[j] = rsqrt(d);
    if (l > j) r[j] *= inv[j];
#pragma unroll
    for (int k = j + 1; k < GE_GROUP; k++) {
      const double lkj = __shfl_sync(gmask, r[j], k, GE_GROUP);  // L[k][j]
      if (l >= k) r[k] -= r[j] * lkj;
    }
  }
  double y = mine ? g_[row] : 0.0;  // L y = g (column oriented): after column j every later row subtracts L[row][j] y_j
#pragma unroll
  for (int j = 0; j < GE_GROUP; j++) {
    const double yj = __shfl_sync(gmask, y, j, GE_GROUP) * inv[j];
    if (l == j) y = yj;
    else if (l > j) y -= r[j] * yj;
  }
#pragma unroll
  for (int i = GE_GROUP - 1; i >= 0; i--) {  // L^T x = y: row l needs L[i][l] (i > l), which lives in lane i's register r[l]
    const double xi = __shfl_sync(gmask, y, i, GE_GROUP) * inv[i];
    double lil = 0.0;
#pragma unroll
    for (int c = 0; c < GE_GROUP; c++) {
      if (c < i) {  // compile-time after unrolling
        const double v = __shfl_sync(gmask, r[c], i, GE_GROUP);
        if (l == c) lil = v;
      }
    }
    if (l == i) y = xi;
    else if (l < i) y -= lil * xi;
  }
  if (mine) x[row] = sign * y;
}

// x := (M + hdamp * diag(damping))^-1 x  for the block-diagonal (per kinematic tree) mass matrix, through dense per-tree
// Cholesky factors in the (currently free) Hessian storage.  Replaces the tree-sparse L^T D L factor/solve when every tree fits
// a lane group; returns false (nothing done) otherwise so that the caller can fall back.
__device__ __noinline__ bool mass_block_solve(double* ws, double* x, double hdamp, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  for (int t = 0; t < m.ntree; t++) if (m.tree_dofnum[t] > GE_GROUP && !m.tree_simple[t]) return false;
  double* H = ws + L.H;
  const double* qM = ws + L.qM;
  // "simple" trees (free-floating single bodies): the block is a model constant, multiply by the precomputed inverse
  // (tree_Minv[t][0] = M^-1, [1] = (M + h*damping)^-1 for h = opt.timestep); results go through a scratch dof vector because every
  // row of a tree reads all of the tree's entries of x
  const int which = hdamp != 0.0 ? 1 : 0;
  double* tmp = ws + L.Mv;  // free dof vector in both callers (before the Newton solve / after it)
  LANE_LOOP(i, m.nv) {
    int t = m.dof_treeindex[i];
    int lo = m.tree_dofadr[t];
    if (m.tree_simple[t]) {
      const double* Mi = m.tree_Minv + ((size_t)(t * 2 + which) * 6 + (i - lo)) * 6;
      double s = 0;
#pragma unroll
      for (int j = 0; j < 6; j++) s += Mi[j] * x[lo + j];
      tmp[i] = s;
    } else {
      // the non-simple trees get their blocks back to back in tree order
      int off = 0;
      for (int u = 0; u < t; u++) if (!m.tree_simple[u]) off += m.tree_dofnum[u] * (m.tree_dofnum[u] + 1) / 2;
      const int r = i - lo;
      double* row = H + off + r * (r + 1) / 2;
      for (int j = 0; j <= r; j++) row[j] = 0;
      int a = m.dof_Madr[i], k = 0;
      for (int j = i; j >= 0; j = m.dof_parentid[j], k++) row[j - lo] = qM[a + k];
      if (hdamp != 0.0) row[r] += hdamp * m.dof_damping[i];
    }
  }
  gsync();
  LANE_LOOP(i, m.nv) if (m.tree_simple[m.dof_treeindex[i]]) x[i] = tmp[i];
  const int g = lane / GE_GROUP, l = lane % GE_GROUP;
  const unsigned gmask = ((1u << GE_GROUP) - 1u) << (((lane & 31) / GE_GROUP) * GE_GROUP);
  // the remaining trees, packed GE_LANES / 8 at a time onto the lane groups
  int slot = 0, off = 0;
  for (int t = 0; t < m.ntree; t++) {
    if (m.tree_simple[t]) continue;
    const int nt = m.tree_dofnum[t];
    if (slot % (GE_LANES / GE_GROUP) == g) group_chol_solve(H + off, m.tree_dofadr[t], nt, l, gmask, x, x, 1.0);
    off += nt * (nt + 1) / 2;
    slot++;
  }
  gsync();
  return true;
}

// x := -H^-1 g.  Uncoupled trees: 8-lane groups (group_chol_solve).  Coupled trees: right-looking dense Cholesky of the island's block
// with one whole warp (each lane owns rows lane, lane+32, ... of the block); the warps of a CTA-per-env build take the islands they
// own (island_owner) concurrently.
__device__ __noinline__ void cholesky_solve(double* ws, int* wi, double* x, const double* g_, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  double* H = ws + L.H;
#if GE_NW > 1
  if (wi[L.i_hflag]) H = g_hovf;
#endif
  const int wl = lane & 31, wid = lane >> 5;
  const int *tcoupled = wi + L.i_tcoupled, *tlist = wi + L.i_tlist;
  bool any_coupled = false;
  for (int t = 0; t < m.ntree; t++) any_coupled |= tcoupled[t] != 0;
  {
    const int g = lane / GE_GROUP, l = lane % GE_GROUP;
    const unsigned gmask = ((1u << GE_GROUP) - 1u) << ((wl / GE_GROUP) * GE_GROUP);
    for (int t0 = 0; t0 < m.ntree; t0 += GE_LANES / GE_GROUP) {
      int t = t0 + g;
      if (t >= m.ntree || tcoupled[t]) continue;  // group-uniform
      group_chol_solve(H + T_HOFF(tlist, t), m.tree_dofadr[t], m.tree_dofnum[t], l, gmask, g_, x, -1.0);
    }
  }
  gsync();
  if (!any_coupled) return;
  // coupled trees: one dense Cholesky per island block (rows in ascending dof order), rows spread over the lanes of the owner warp.
  // The block-row -> dof lists of the islands are laid out one after the other in the int scratch (the islands partition the
  // coupled trees).
  const int* island = wi + L.i_island;
  int* idx_all = (int*)wi + L.i_first;  // (the row-envelope array of the skyline version; free here)
  int idx_off = 0;
  for (int rep = 0; rep < m.ntree; rep++) {
    if (!tcoupled[rep] || island[rep] != rep) continue;
    const int n = tlist[rep * GE_TLIST];  // island size, recorded by build_hessian
    int* idx = idx_all + idx_off;
    idx_off += n;
    if (GE_NW > 1 && island_owner(island, tlist, rep) != wid) continue;
    double* Hb = H + T_HOFF(tlist, rep);
    {
      int r0 = 0;
      for (int t = rep; t < m.ntree; t++) {
        if (!tcoupled[t] || island[t] != rep) continue;
        int lo = m.tree_dofadr[t], nt = m.tree_dofnum[t];
        for (int k = wl; k < nt; k += 32) idx[r0 + k] = lo + k;
        r0 += nt;
      }
    }
    __syncwarp();
    for (int j = 0; j < n; j++) {
      double d = Hb[HIDX(j, j)];
      if (d < GE_MINVAL) d = GE_MINVAL;
      const double ljj = sqrt(d), inv = 1.0 / ljj;
      __syncwarp();
      for (int i = j + 1 + wl; i < n; i += 32) Hb[HIDX(i, j)] *= inv;
      if (wl == 0) Hb[HIDX(j, j)] = ljj;
      __syncwarp();
      for (int i = j + 1 + wl; i < n; i += 32) {
        const double lij = Hb[HIDX(i, j)];
        if (lij == 0.0) continue;
        double* row = Hb + HIDX(i, 0);
        for (int k = j + 1; k <= i; k++) row[k] -= lij * Hb[HIDX(k, j)];
      }
      __syncwarp();
    }
    for (int i = wl; i < n; i += 32) x[idx[i]] = g_[idx[i]];
    __syncwarp();
    for (int j = 0; j < n; j++) {  // L y = g, column oriented
      const int dj = idx[j];
      double yj = x[dj] / Hb[HIDX(j, j)];
      __syncwarp();
      if (wl == 0) x[dj] = yj;
      for (int i = j + 1 + wl; i < n; i += 32) x[idx[i]] -= Hb[HIDX(i, j)] * yj;
      __syncwarp();
    }
    for (int i = n - 1; i >= 0; i--) {  // L^T x = y, column oriented
      const int di = idx[i];
      double xi = x[di] / Hb[HIDX(i, i)];
      __syncwarp();
      if (wl == 0) x[di] = xi;
      const double* row = Hb + HIDX(i, 0);
      for (int k = wl; k < i; k += 32) x[idx[k]] -= row[k] * xi;
      __syncwarp();
    }
    for (int i = wl; i < n; i += 32) x[idx[i]] = -x[idx[i]];
    __syncwarp();
  }
  gsync();
}

}  // namespace ge
