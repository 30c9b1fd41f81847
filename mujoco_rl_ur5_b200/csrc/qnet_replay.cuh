// Prioritized experience replay for the online trainer (Schaul et al. 2016, "Prioritized Experience Replay", proportional variant):
// a device sum-tree over the replay slots, stratified proportional sampling with importance weights, and the priority update.
//
// Tree: an implicit binary heap of 2 cap doubles, cap = the smallest power of two >= the replay size.  Slot i is leaf cap + i, node k
// has children 2k and 2k + 1, the root tree[1] holds the total (tree[0] is unused).  Every internal node is recomputed as the sum of its
// two children after a leaf changes (never updated by adding deltas), so the tree cannot drift and its contents are a function of the
// leaves alone.  Leaves of slots never filled are 0.  pmax (one device double, 1.0 at the start) is the largest priority ever assigned.
//
// The three kernels are single-CTA: a push touches a few thousand leaves once per batched step, a sample / update B = 12 leaves at
// a tree depth of about 20, so the work is a chain of dependent loads per thread and one CTA with __syncthreads between tree levels
// is all the parallelism there is to use.
// Included at the end of qnet.cu (same library, C-ABI in include/grasp_qnet.h).
#pragma once

#define PER_C0 0xC0000000u  // counter domain of the stratum draws (the keyed-draw table above keyed_words in qnet.cu)
#define PER_THREADS 1024

// max of one double per thread over the CTA; every thread gets the result
__device__ __forceinline__ double per_block_max(double v, double* sred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  if (lane == 0) sred[warp] = v;
  __syncthreads();
  v = lane < nw ? sred[lane] : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// New transitions: leaves of the n claimed slots := pmax, then their ancestors level by level.  A push claims consecutive ring
// slots, so neighbours share ancestors: of a run of entries with the same node at a level only the first recomputes it.
__global__ void __launch_bounds__(PER_THREADS) k_per_push(double* __restrict__ tree, const double* __restrict__ pmax, const long long* __restrict__ slot, int n,
                                                          long long cap, int levels) {
  const double pm = *pmax;
  for (int i = threadIdx.x; i < n; i += blockDim.x) tree[cap + slot[i]] = pm;
  for (int l = 1; l <= levels; l++) {
    __syncthreads();  // level l - 1 complete (global writes of the CTA are visible after the barrier)
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const long long node = (cap + slot[i]) >> l;
      if (i > 0 && ((cap + slot[i - 1]) >> l) == node) continue;
      tree[node] = tree[2 * node] + tree[2 * node + 1];
    }
  }
}

// Stratum j < B: U = 53-bit uniform of the keyed draw (PER_C0 + j, update, rank) under seed, u = (j + U) total / B, then the descent
// from the root: right iff u >= left and the right subtree holds mass (u -= left), else left.  Every node reached has a positive sum
// (it is the root, or a child chosen for being positive, or the left child of a node whose right child is 0), so the walk never ends
// on an empty leaf, even where rounding puts u at or past the total.  Importance weight (length p / total)^-beta over the batch's
// largest, in double, stored as f32.
__global__ void __launch_bounds__(PER_THREADS) k_per_sample(const double* __restrict__ tree, long long cap, long long length, int B, double beta,
                                                            unsigned long long seed, unsigned long long update, unsigned int rank, long long* __restrict__ idx_out,
                                                            float* __restrict__ w_out) {
  __shared__ double sred[32];
  const int j = threadIdx.x;
  const double total = tree[1];
  double w = 0.0;
  if (j < B) {
    uint32_t r[4];
    philox4x32_10(PER_C0 + (uint32_t)j, (uint32_t)update, (uint32_t)(update >> 32), rank, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const double U = (double)((((uint64_t)(r[0] >> 5)) << 26) + (uint64_t)(r[1] >> 6)) * 0x1p-53;
    double u = ((double)j + U) * (total / (double)B);
    long long node = 1;
    while (node < cap) {
      const double left = tree[2 * node], right = tree[2 * node + 1];
      if (u >= left && right > 0.0) { u -= left; node = 2 * node + 1; }
      else node = 2 * node;
    }
    idx_out[j] = node - cap;
    w = pow((double)length * tree[node] / total, -beta);
  }
  const double wmax = per_block_max(w, sred);
  if (j < B) w_out[j] = (float)(w / wmax);
}

// Priorities of a trained batch: p_j = (|r_j - q_j| + eps)^alpha, r_j the training target (the reward at gamma = 0, the Bellman target
// y with bootstrapping), so |r_j - q_j| is the TD error.  Leaves are written in batch order - of a slot drawn more than once only the
// last entry writes - and then every entry walks its ancestors, one level per barrier (entries sharing a node write the same sum).  pmax := max(pmax, max_j p_j).
__global__ void __launch_bounds__(PER_THREADS) k_per_update(double* __restrict__ tree, double* __restrict__ pmax, const long long* __restrict__ idx,
                                                            const float* __restrict__ qsel, const float* __restrict__ reward, int B, double alpha, double eps,
                                                            long long cap, int levels) {
  __shared__ double sred[32];
  const int j = threadIdx.x;
  long long node = 0;
  double p = 0.0;
  if (j < B) {
    p = pow(fabs((double)reward[j] - (double)qsel[j]) + eps, alpha);
    const long long s = idx[j];
    bool last = true;
    for (int k = j + 1; k < B; k++) last = last && idx[k] != s;
    node = cap + s;
    if (last) tree[node] = p;
  }
  const double m = per_block_max(p, sred);
  if (j == 0 && m > *pmax) *pmax = m;
  for (int l = 0; l < levels; l++) {
    __syncthreads();
    if (j < B) {
      node >>= 1;
      tree[node] = tree[2 * node] + tree[2 * node + 1];
    }
  }
}

// ------------------------------------------------------------------------------------------------ C-ABI
static int per_levels(int cap) {  // log2(cap); -1 unless cap is a power of two in [1, 2^30]
  if (cap <= 0 || cap > (1 << 30) || (cap & (cap - 1))) return -1;
  int l = 0;
  while ((1 << l) < cap) l++;
  return l;
}
extern "C" int gq_per_push(double* tree, const double* pmax, const long long* slot, int n, int cap, void* stream) {
  const int levels = per_levels(cap);
  if (!tree || !pmax || (n > 0 && !slot) || n < 0 || n > cap || levels < 0) { snprintf(q_err, sizeof q_err, "gq_per_push: bad argument"); return -1; }
  if (n == 0) return 0;
  k_per_push<<<1, PER_THREADS, 0, (cudaStream_t)stream>>>(tree, pmax, slot, n, (long long)cap, levels);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_per_sample(const double* tree, int cap, long long length, int B, double beta, unsigned long long seed, unsigned long long update,
                             unsigned int rank, long long* idx_out, float* weight_out, void* stream) {
  if (!tree || !idx_out || !weight_out || per_levels(cap) < 0 || length <= 0 || length > cap || B <= 0 || B > PER_THREADS || !(beta >= 0.0)) {
    snprintf(q_err, sizeof q_err, "gq_per_sample: bad argument");
    return -1;
  }
  k_per_sample<<<1, (B + 31) & ~31, 0, (cudaStream_t)stream>>>(tree, (long long)cap, length, B, beta, seed, update, rank, idx_out, weight_out);
  QCK(cudaGetLastError());
  return 0;
}
extern "C" int gq_per_update(double* tree, double* pmax, const long long* idx, const float* qsel, const float* reward, int B, double alpha, double eps, int cap,
                             void* stream) {
  const int levels = per_levels(cap);
  if (!tree || !pmax || !idx || !qsel || !reward || B <= 0 || B > PER_THREADS || !(alpha >= 0.0) || !(eps >= 0.0) || levels < 0) {
    snprintf(q_err, sizeof q_err, "gq_per_update: bad argument");
    return -1;
  }
  k_per_update<<<1, (B + 31) & ~31, 0, (cudaStream_t)stream>>>(tree, pmax, idx, qsel, reward, B, alpha, eps, (long long)cap, levels);
  QCK(cudaGetLastError());
  return 0;
}
