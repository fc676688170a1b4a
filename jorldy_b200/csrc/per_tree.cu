// Prioritised-replay sum-tree kept resident in HBM (float64 array heap), batched update /
// store / sample kernels with the reference's *sequential* semantics reproduced bit-for-bit.
//
// Replaces jorldy/core/buffer/per_buffer.py:
//   :19-40  store / add_tree_data      -> jb_per_update on a run of consecutive leaves
//   :42-54  update_priority/update_tree -> jb_per_update
//   :56-68  search_tree                 -> descent inside jb_per_sample
//   :70-101 sample (uniform/prioritised split, IS weights, stats) -> jb_per_sample
//
// Tree layout is the reference's: tree_size = 2N-1, root at 0, children 2i+1 / 2i+2, leaves at
// N-1 .. 2N-2, float64.  (1 M slots -> 16 MB, 2 M -> 32 MB: L2-resident in H100's 50 MB L2.)
//
// Bit-exactness of the incremental-delta tree (SURVEY hard part 2): the reference applies a
// batch of B updates one after another, each adding delta_i = new_i - old_i to every ancestor.
// f64 addition does not commute in rounding, but additions to *different* nodes are
// independent, so we parallelise over tree nodes instead of over updates: for every distinct
// ancestor touched by the batch exactly one thread ("owner" = the first batch entry that reaches
// the node) walks the batch in order and adds the deltas of the entries below that node, in the
// reference's order.  Duplicate leaves inside a batch are honoured (old_i of a later duplicate
// is the earlier duplicate's new value; last write wins), exactly as the python loop
// (rainbow.py:230-231, ape_x.py:111-112) behaves.
#include "common.cuh"
#include "philox.cuh"

namespace {

__device__ __forceinline__ bool is_proper_ancestor(uint32_t a_plus1, uint32_t x_plus1) {
  int da = 32 - __clz(a_plus1), dx = 32 - __clz(x_plus1);
  if (dx <= da) return false;
  return (x_plus1 >> (dx - da)) == a_plus1;
}

// ---- sampling -------------------------------------------------------------------------------
// One CTA; thread per sample slot (strided when B > blockDim).  Output order follows the
// reference: the K uniformly-drawn slots first, then the B-K prioritised ones (per_buffer.py:84).
// u_a[B], u_b[B]: uniforms in [0,1); slot s is "uniform" iff it is among the first K = #{u_a < usp}
// slots, uses floor(u_b[s]*counter) as ring index if uniform, u_b[s]*total as descent target otherwise.
__global__ void __launch_bounds__(512) per_sample_kernel(const double* __restrict__ tree, int64_t first_leaf, int64_t counter,
                                  int B, double beta, double usp, const double* __restrict__ u_a,
                                  const double* __restrict__ u_b, uint64_t seed, uint64_t rng_ctr,
                                  const double* __restrict__ shard_prob, const int64_t* __restrict__ global_counter,
                                  int64_t* __restrict__ out_idx, double* __restrict__ out_w,
                                  double* __restrict__ out_p, double* __restrict__ out_stats, int normalize) {
  __shared__ int s_count;
  __shared__ double s_red[32];
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  // K = number of uniform slots
  int local = 0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    double ua;
    if (u_a) ua = u_a[i];
    else { jb_philox4 r = jb_philox(seed, (uint64_t)i, rng_ctr); ua = jb_u01_double(r.x, r.y); }
    if (ua < usp) ++local;
  }
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(&s_count, local);
  __syncthreads();
  const int K = s_count;
  const double total = tree[0];
  // Sharded replay: this tree is one of G shards and receives a 1/G share of every batch, so item i of this shard is
  // drawn with probability shard_prob * [(1-usp) p_i / total_local + usp / count_local]  (shard_prob = 1/G), while the
  // uniform reference probability of the importance weight is 1 / N_global (per_buffer.py:88-93 over the union).
  const double shard_p = shard_prob ? *shard_prob : 1.0;
  const double cnt_global = (double)(global_counter ? *global_counter : counter);

  double wmax = 0.0, psum = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    double ub;
    if (u_b) ub = u_b[i];
    else { jb_philox4 r = jb_philox(seed, (uint64_t)i, rng_ctr); ub = jb_u01_double(r.z, r.w); }
    int64_t idx;
    if (i < K) {
      int64_t r = (int64_t)(ub * (double)counter);
      if (r >= counter) r = counter - 1;
      idx = r + first_leaf;
    } else {
      double num = __dmul_rn(ub, total);
      idx = 0;
      while (idx < first_leaf) {            // per_buffer.py:56-68
        const int64_t left = 2 * idx + 1;
        const double lv = tree[left];
        if (num <= lv) idx = left;
        else { num = __dadd_rn(num, -lv); idx = left + 1; }
      }
    }
    const double p = tree[idx];
    // per_buffer.py:88-93
    const double uniform_prob = 1.0 / (double)counter;
    const double prio_prob = p / total;
    double sample_prob = __dadd_rn(__dmul_rn(1.0 - usp, prio_prob), __dmul_rn(usp, uniform_prob));
    double ref_prob = uniform_prob;
    if (shard_prob) { sample_prob = __dmul_rn(shard_p, sample_prob); ref_prob = 1.0 / cnt_global; }
    const double w = pow(ref_prob / sample_prob, beta);
    out_idx[i] = idx; out_p[i] = p; out_w[i] = w;
    wmax = fmax(wmax, w); psum += p;
  }
  // block reductions (max weight, sum of sampled priorities)
  for (int o = 16; o > 0; o >>= 1) wmax = fmax(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = wmax;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < (blockDim.x + 31) / 32 ? s_red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (threadIdx.x == 0) s_red[0] = v;
  }
  __syncthreads();
  wmax = s_red[0];
  __syncthreads();
  psum = jb_warp_sum_d(psum);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = psum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) s += s_red[w];
    out_stats[0] = s / (double)B;                 // sampled_p = mean(priorities)
    out_stats[1] = total / (double)counter;       // mean_p
    out_stats[2] = wmax;                          // max raw IS weight (for sharded normalisation)
    out_stats[3] = (double)K;
  }
  if (normalize)
    for (int i = threadIdx.x; i < B; i += blockDim.x) out_w[i] = out_w[i] / wmax;
}

__global__ void per_scale_weights_kernel(double* __restrict__ w, const double* __restrict__ wmax, int B) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) w[i] = w[i] / *wmax;
}

// Internal levels: grid.x = k-1 for the k-th ancestors (k >= 1); block = threads over the batch.
// These blocks only *read* leaves (to form delta_i); the leaves themselves are rewritten by a
// second launch (per_update_leaves_kernel) ordered after this one on the stream.
// dynamic smem: double delta[B]; double new[B]; int32 leaf[B]
__global__ void per_update_levels_kernel(double* __restrict__ tree, const int64_t* __restrict__ tree_idx,
                                         int64_t first_idx, int64_t tree_size, int64_t first_leaf,
                                         const double* __restrict__ new_p, const double* __restrict__ fill_p,
                                         int B) {
  extern __shared__ unsigned char smem_raw[];
  double* s_delta = reinterpret_cast<double*>(smem_raw);
  double* s_new = s_delta + B;
  int32_t* s_leaf = reinterpret_cast<int32_t*>(s_new + B);
  const int k = blockIdx.x + 1;
  const double fill = fill_p ? *fill_p : 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    int64_t li;
    if (tree_idx) li = tree_idx[i];
    else {
      li = first_idx + i;
      const int64_t n_leaf = tree_size - first_leaf;
      if (li >= tree_size) li = first_leaf + (li - first_leaf) % n_leaf;
    }
    s_leaf[i] = (int32_t)li;
    s_new[i] = new_p ? new_p[i] : fill;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const int32_t li = s_leaf[i];
    double old_v = 0.0; bool found = false;
    for (int j = i - 1; j >= 0; --j) if (s_leaf[j] == li) { old_v = s_new[j]; found = true; break; }
    if (!found) old_v = tree[li];
    s_delta[i] = __dadd_rn(s_new[i], -old_v);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const uint32_t x = (uint32_t)s_leaf[i] + 1u;
    const uint32_t a1 = x >> k;
    if (a1 == 0) continue;
    bool owner = true;
    for (int j = 0; j < i; ++j) if (is_proper_ancestor(a1, (uint32_t)s_leaf[j] + 1u)) { owner = false; break; }
    if (!owner) continue;
    double acc = tree[a1 - 1];
    for (int j = i; j < B; ++j)
      if (is_proper_ancestor(a1, (uint32_t)s_leaf[j] + 1u)) acc = __dadd_rn(acc, s_delta[j]);
    tree[a1 - 1] = acc;
  }
}

__global__ void per_update_leaves_kernel(double* __restrict__ tree, const int64_t* __restrict__ tree_idx,
                                         int64_t first_idx, int64_t tree_size, int64_t first_leaf,
                                         const double* __restrict__ new_p, const double* __restrict__ fill_p,
                                         double* __restrict__ max_priority, int B) {
  extern __shared__ unsigned char smem_raw[];
  double* s_new = reinterpret_cast<double*>(smem_raw);
  int32_t* s_leaf = reinterpret_cast<int32_t*>(s_new + B);
  __shared__ double s_mx[32];
  const double fill = fill_p ? *fill_p : 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    int64_t li;
    if (tree_idx) li = tree_idx[i];
    else {
      li = first_idx + i;
      const int64_t n_leaf = tree_size - first_leaf;
      if (li >= tree_size) li = first_leaf + (li - first_leaf) % n_leaf;
    }
    s_leaf[i] = (int32_t)li;
    s_new[i] = new_p ? new_p[i] : fill;
  }
  __syncthreads();
  double mx = -1.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const int32_t li = s_leaf[i];
    bool last = true;
    for (int j = i + 1; j < B; ++j) if (s_leaf[j] == li) { last = false; break; }
    if (last) tree[li] = s_new[i];
    mx = fmax(mx, s_new[i]);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_mx[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = *max_priority;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) m = fmax(m, s_mx[w]);
    *max_priority = m;
  }
}

__global__ void per_rebuild_level_kernel(double* __restrict__ tree, int64_t lo, int64_t hi) {
  int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < hi) tree[i] = __dadd_rn(tree[2 * i + 1], tree[2 * i + 2]);
}

}  // namespace

static int per_levels(int64_t tree_size) {
  int d = 0; int64_t x = tree_size;   // 1-based id of the last node
  while (x > 1) { x >>= 1; ++d; }
  return d;                           // max number of proper ancestors of any leaf
}

// Apply B priority writes with the reference's sequential semantics.
//   tree_idx  : [B] int64 tree coordinates (>= capacity-1) or NULL for the consecutive run starting
//               at `first_idx` (the PERBuffer.store path; wraps from tree_size to first_leaf)
//   new_p     : [B] f64 priorities or NULL -> every write uses *fill_p (PERBuffer.max_priority)
//   max_priority : device f64 scalar, updated to max(old, all new)       (per_buffer.py:48)
JB_API int jb_per_update(double* tree, int64_t capacity, const int64_t* tree_idx, int64_t first_idx,
                         const double* new_p, const double* fill_p, double* max_priority, int B,
                         void* stream) {
  if (!tree || capacity <= 0 || B <= 0 || !max_priority) return JB_ERR_INVALID;
  if (!new_p && !fill_p) return JB_ERR_INVALID;
  if (B > 8192) return JB_ERR_INVALID;   // host wrapper splits larger batches (sequential semantics allow it)
  const int64_t tree_size = 2 * capacity - 1, first_leaf = capacity - 1;
  cudaStream_t s = (cudaStream_t)stream;
  const int levels = per_levels(tree_size);
  const int threads = B >= 256 ? 256 : ((B + 31) / 32) * 32;
  size_t smem = (size_t)B * (8 + 8 + 4);
  if (smem > 48 * 1024) {
    cudaFuncSetAttribute(per_update_levels_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(per_update_leaves_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  if (levels > 0)
    per_update_levels_kernel<<<levels, threads, smem, s>>>(tree, tree_idx, first_idx, tree_size, first_leaf, new_p, fill_p, B);
  per_update_leaves_kernel<<<1, threads, (size_t)B * 12, s>>>(tree, tree_idx, first_idx, tree_size, first_leaf, new_p, fill_p,
                                                            max_priority, B);
  return jb_check_launch();
}

// Draw B tree indices + importance weights.  u_a/u_b NULL -> Philox(seed, slot, rng_ctr).
// out_stats[4] = {sampled_p, mean_p, max raw weight, #uniform slots}.
// shard_prob/global_counter (device scalars, may be NULL): when the tree is one shard of a multi-GPU replay the
// sampling probability is shard_prob x the local one and the weight's reference probability is
// 1 / global_counter; with normalize=0 the raw
// weights are returned so the caller can divide by the all-reduced max (jb_per_scale_weights).
JB_API int jb_per_sample(const double* tree, int64_t capacity, int64_t counter, int B, double beta,
                         double uniform_sample_prob, const double* u_a, const double* u_b, uint64_t seed,
                         uint64_t rng_ctr, const double* shard_prob, const int64_t* global_counter,
                         int64_t* out_idx, double* out_w, double* out_p, double* out_stats, int normalize,
                         void* stream) {
  if (!tree || capacity <= 0 || counter <= 0 || B <= 0 || !out_idx || !out_w || !out_p || !out_stats)
    return JB_ERR_INVALID;
  const int threads = B >= 512 ? 512 : ((B + 31) / 32) * 32;
  per_sample_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(tree, capacity - 1, counter, B, beta, uniform_sample_prob,
                                                             u_a, u_b, seed, rng_ctr, shard_prob, global_counter,
                                                             out_idx, out_w, out_p, out_stats, normalize);
  return jb_check_launch();
}

JB_API int jb_per_scale_weights(double* w, const double* wmax, int B, void* stream) {
  if (!w || !wmax || B <= 0) return JB_ERR_INVALID;
  per_scale_weights_kernel<<<jb_div_up(B, 256), 256, 0, (cudaStream_t)stream>>>(w, wmax, B);
  return jb_check_launch();
}

// Recompute every internal node from its children (bottom-up, one launch per level). Not part of
// the reference's behaviour (its tree is only ever delta-updated); provided for checkpoint restore
// and for tests that want an exactly-summed tree.
JB_API int jb_per_rebuild(double* tree, int64_t capacity, void* stream) {
  if (!tree || capacity <= 0) return JB_ERR_INVALID;
  const int64_t first_leaf = capacity - 1;
  // internal nodes are [0, first_leaf); heap level d spans [2^d - 1, 2^(d+1) - 1)
  int dmax = 0;
  while ((((int64_t)1) << (dmax + 1)) - 1 < first_leaf) ++dmax;
  for (int d = dmax; d >= 0; --d) {
    int64_t lo = (((int64_t)1) << d) - 1, hi = (((int64_t)1) << (d + 1)) - 1;
    if (hi > first_leaf) hi = first_leaf;
    if (lo >= hi) continue;
    per_rebuild_level_kernel<<<jb_div_up(hi - lo, 256), 256, 0, (cudaStream_t)stream>>>(tree, lo, hi);
  }
  return jb_check_launch();
}
