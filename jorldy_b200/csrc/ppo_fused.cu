// Persistent cooperative kernel: a whole run of PPO minibatch steps (ppo.py:118-175 — forward, clipped
// surrogate / clipped value / entropy loss, backward, global-norm clip, Adam) in ONE launch.
//
// Why: at the reference's minibatch size (256 x [4-512-512-(A+1)]) one step is ~0.4 GFLOP and < 4 MB of
// traffic, i.e. microseconds of work, and one learn() is n_epoch * N*T/B = 6144 strictly sequential
// steps.  As 13 separate launches per step (the "graph" path) almost all of a step is launch gaps and
// cold per-kernel load latency.  Here one CTA per SM stays resident for the whole epoch and a step is
// THREE phases separated by a hand-rolled grid barrier (scripts/bench_gridbar.cu compares the variants):
//
//   P1  layer-2 forward tiles (32x32, fp32 FFMA, 16-way in-CTA split-K).  The A panel h1 = relu(x W1^T + b1)
//       is GENERATED in shared memory from the gathered state rows (K = D <= 16), never read from HBM; the
//       W2 panel arrives by cp.async.cg.  The epilogue also emits, per tile, the PARTIAL head outputs
//       sum_{n in tile} h2[m, n] Wh[o, n], so that nobody has to re-read h2 rows to evaluate the heads.
//       Every finished tile draws a ticket of its row tile; the CTA that draws the last one folds the row tile's
//       partial head outputs and runs the loss row maths (ppo_rowmath.cuh, one thread per row) ONCE for those
//       rows, into per-row tables in L2 (d loss/d head outputs, per-row statistics) that the barrier publishes.
//   P3  critic means + backward.  Every CTA bulk-copies the d loss/d head outputs of the minibatch into shared
//       memory and folds the per-row statistics into the two critic means.  Then the backward jobs, each with
//       its panels prefetched while the previous job reduces (the first JB job's W2t panel before the barrier):
//         JB  dh1 tile = ((dout Wh) * relu'(h2)) W2, masked by relu'(h1); dh2 is generated in place in the
//             A panel; the epilogue turns the tile into PARTIAL dW1/db1 (x rows are <= 64 B each), so dh1
//             never leaves the SM.
//         JA  a PAIR of dW2 tiles sharing one generated dh2 panel (+ db2 as the panel row-sum).
//         JC  head weight / bias gradients, 32 columns per job.
//         JD  fixed-order fold of the MT partial dW1/db1 (waits on a per-column-tile completion counter
//             that the JB jobs bump — every CTA runs its JB jobs first, so the wait cannot deadlock).
//       Every job adds its outputs' squares to a per-thread accumulator; one block reduction per step
//       publishes the CTA's share of ||g||^2.
//   P5  Adam on a static 1/gridDim slice of the flat parameter buffer; p/m/v of the slice are loaded into
//       registers BEFORE the barrier, the clip coefficient comes from a fixed-order fold of the partials.
//
// Determinism: static job -> CTA maps, fixed-order reductions, no float atomics: bit-reproducible run
// to run.  Coherence: every buffer written inside the kernel is read with ld.global.cg / cp.async.cg
// (L2), and the barrier's gpu-scope release/acquire orders the phases.
//
// Multi-GPU (args.world > 1): every rank's flat gradient lives in a peer-mapped exchange buffer (args.peer[r],
// torch symmetric memory) and the gradient average is a reduce-scatter + all-gather done by the kernel itself in
// "LL" words: every 32-bit datum crosses NVLink as one aligned 64-bit word {step tag | value}, which is valid exactly
// when its tag equals the step number (64-bit stores are single-copy atomic) — no flags, no fences, one NVLink traversal
// per hop.  After the backward phase's barrier
//   * every CTA pushes its chunk of every other rank's slice of the local gradient into that owner's inbox;
//   * rank q OWNS slice q, CTA c of rank q chunk c of it: it sums the ranks' copies in rank order, scales by 1/world,
//     pushes the averaged chunk into EVERY rank's copy of the averaged gradient and the chunk's squared norm into every
//     rank's norm table;
//   * every CTA reads its Adam slice of the averaged gradient and all chunk norms as they arrive, folds the norms in a
//     fixed order (identical bits on all ranks) and applies clip + Adam.
//   Flag + fence protocols were slower: every hop paid a release store or system fence waiting for remote write
//   acknowledgements plus acquire polls, and un-throttled relaxed polling of flags saturated L2.
//   * the two scalar means of critic_loss = max(mean, mean) (ppo.py:151-154) are GLOBAL: each rank sends its two row sums to
//     the peers right after bar1 (two LL words); receiving step s's message from a peer also proves that the peer has
//     finished step s-1.
// No NCCL call between backward and Adam.
//
// Constraints (else the host uses the multi-launch path): B % 32 == 0, B <= 512, H % 32 == 0, H <= 512,
// D <= 16, nout <= 8; multi-GPU additionally: <= 8 ranks.
#include <cstdlib>
#include "common.cuh"
#include "ppo_rowmath.cuh"
#include "wgmma.cuh"
#include "../../include/jorldy_b200_fused.h"

namespace {

constexpr int NT = 256;
constexpr int PK = 512;
constexpr int MAXD = 16;
constexpr int MAXO = 8;
constexpr int KG = 16;                                  // in-CTA split-K groups
constexpr int SMALL_FLOATS = 2048;                      // xs[32*16], reduction scratch, row ids
constexpr int RED_FLOATS = KG * (32 * 36 + 16);   /* = KG * RED_GS */         // 18688: split-K fold area; also >= a 32x(PK+4) or PKx36 panel
constexpr int JA_ROWS = 256;                            // minibatch rows per dW2 / head-gradient panel
constexpr int R2_FLOATS = JA_ROWS * 32;                 // 8192: a dense [256][32] panel
constexpr int MAX_B = 512;                              // minibatch rows (row-phase scratch in s_small)
constexpr int ADAM_IT = 4;                              // float4 per thread kept in registers across the barrier
constexpr int PS_FLOATS = (MAXO + 2) * PK;                // per-CTA parameter stash: head rows [MAXO][PK], b2, b1
constexpr int CTR_ROW = 1;                              // a.barrier[CTR_ROW + mt]: finished P1 tiles of row tile mt (tickets)
constexpr int CTR_JB = 32;                              // a.barrier[CTR_JB + kt]: finished JB jobs of column tile kt

typedef jb_ppo_fused_args Args;

__device__ __forceinline__ float ldcg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

// ---- panel staging: TMA 1-D bulk copies (cp.async.bulk, one request per panel row) completing on one
// mbarrier.  (The first versions issued 16-byte cp.async per thread: 4-8 K LDGSTS per panel fill the SM's
// load queue, so "prefetching" stalled the issuing warps for as long as the transfer took and every
// ordinary load behind them waited too.  A bulk request costs one instruction per 128 B - 2 KB row and
// the copy engine does the rest.)  Exactly one group of copies is in flight at a time: `Stager` tracks
// the bytes of the group being issued and the phase parity of the barrier.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
// one 4-byte word global -> shared without a register: data fetched a whole tile ahead of its use
__device__ __forceinline__ void cp_async4(float* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
struct Stager {
  unsigned mbar;      // shared-space address of the mbarrier
  unsigned bytes;     // bytes issued in the open group (uniform across the CTA)
  unsigned parity;    // phase parity the next wait() completes on
  __device__ __forceinline__ void init(void* bar) {
    mbar = smem_u32(bar); bytes = 0; parity = 0;
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(mbar) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
  }
  __device__ __forceinline__ void copy(void* dst, const void* src, unsigned nbytes) const {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(nbytes), "r"(mbar) : "memory");
  }
  __device__ __forceinline__ void commit() {
    if (bytes && threadIdx.x == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(mbar), "r"(bytes) : "memory");
    bytes = 0;
  }
  __device__ __forceinline__ void wait() {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(mbar), "r"(parity)
        : "memory");
    parity ^= 1u;
  }
};

// ---- cross-GPU waits (multi-GPU gradient exchange) are bounded in time (a peer may legitimately be seconds late: it is
// another process with its own host-side launch sequence), and once one wait has given up every later wait returns at once
// (`abort_flag`, a word of this GPU's barrier block), so that a dead peer costs one time-out per launch instead of one per
// step; the host then raises (ppo.py checks acc[7]).  Time = SM cycles (clock64: a register read; %globaltimer costs
// microseconds per read).
constexpr long long X_TIMEOUT_CYCLES = 60ll * 1965000000ll;   // ~60 s of SM clock (clock64: a register read)
constexpr int CTR_ABORT = 63;                           // a.barrier[CTR_ABORT] != 0: an exchange wait timed out
// ---- "LL" words (NCCL's low-latency idea): every 32-bit datum travels as one aligned 64-bit word {tag | value}; an aligned 64-bit
// store is single-copy atomic, so a word whose tag equals the step number carries a valid value — no flag, no fence, no
// ordering between different words is needed, and the latency of an exchange hop is one NVLink traversal.
__device__ __forceinline__ unsigned long long ll_pack(float v, unsigned int tag) {
  return ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
}
__device__ __forceinline__ void ll_store4(unsigned long long* dst /* 4 words, 32-byte aligned */, float4 v, unsigned int tag) {
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};\n" ::"l"(dst), "l"(ll_pack(v.x, tag)), "l"(ll_pack(v.y, tag)) : "memory");
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};\n" ::"l"(dst + 2), "l"(ll_pack(v.z, tag)), "l"(ll_pack(v.w, tag)) : "memory");
}
// spins until the four words at src carry `tag`; false after the exchange time-out (or once another wait has given up)
__device__ __forceinline__ bool ll_load4(const unsigned long long* src, unsigned int tag, float4& v, unsigned int* abort_flag) {
  unsigned long long w0, w1, w2, w3;
  const long long t0 = clock64();
  for (int it = 0;; ++it) {
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];\n" : "=l"(w0), "=l"(w1) : "l"(src) : "memory");
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];\n" : "=l"(w2), "=l"(w3) : "l"(src + 2) : "memory");
    if ((unsigned int)(w0 >> 32) == tag && (unsigned int)(w1 >> 32) == tag && (unsigned int)(w2 >> 32) == tag && (unsigned int)(w3 >> 32) == tag) break;
    if ((it & 63) == 63) {
      unsigned int ab;
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(ab) : "l"(abort_flag) : "memory");
      if (ab || clock64() - t0 > X_TIMEOUT_CYCLES) {
        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;\n" ::"l"(abort_flag), "r"(1u) : "memory");
        v = make_float4(0.f, 0.f, 0.f, 0.f);
        return false;
      }
    }
  }
  v = make_float4(__uint_as_float((unsigned int)w0), __uint_as_float((unsigned int)w1), __uint_as_float((unsigned int)w2), __uint_as_float((unsigned int)w3));
  return true;
}
__device__ __forceinline__ bool ll_load1(const unsigned long long* src, unsigned int tag, float& v, unsigned int* abort_flag) {
  unsigned long long w;
  const long long t0 = clock64();
  for (int it = 0;; ++it) {
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];\n" : "=l"(w) : "l"(src) : "memory");
    if ((unsigned int)(w >> 32) == tag) break;
    if ((it & 63) == 63) {
      unsigned int ab;
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(ab) : "l"(abort_flag) : "memory");
      if (ab || clock64() - t0 > X_TIMEOUT_CYCLES) {
        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;\n" ::"l"(abort_flag), "r"(1u) : "memory");
        v = 0.f;
        return false;
      }
    }
  }
  v = __uint_as_float((unsigned int)w);
  return true;
}

// ---- grid barrier (all CTAs co-resident: cooperative launch) ------------------------------------------
__device__ __forceinline__ void grid_bar(unsigned int* ctr, unsigned int& epoch, unsigned int nctas) {
  __syncthreads();                       // CTA scope: every thread's phase writes happen-before thread 0's release
  if (threadIdx.x == 0) {
    epoch += 1;
    const unsigned int target = epoch * nctas;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(ctr) : "memory");
    unsigned int v;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(ctr) : "memory");
    } while (v < target);
    asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    asm volatile("fence.proxy.async;\n" ::: "memory");   // other SMs' generic-proxy writes before this SM's bulk copies
  }
  __syncthreads();
}

// k-contiguous panel with padded rows: sm[r*(kp+4) + k] = G[(r0+r)*ld + k0 + k], r < 32, k < kp
// (32 requests of kp*4 bytes, one lane of every 8)
__device__ __forceinline__ void stage_kc(Stager& st, float* sm, const float* G, int ld, int r0, int k0, int kp) {
  if ((threadIdx.x & 7) == 0) {
    const int row = threadIdx.x >> 3;
    st.copy(&sm[row * (kp + 4)], &G[(size_t)(r0 + row) * ld + k0], (unsigned)kp * 4u);
  }
  st.bytes += 32u * (unsigned)kp * 4u;
}
// dense [rows][32] panel that is ONE contiguous block in global memory (the tiled h1t / h2t / W2t layouts)
__device__ __forceinline__ void stage_block(Stager& st, float* sm, const float* G, int rows) {
  if (threadIdx.x == 0) st.copy(sm, G, (unsigned)rows * 128u);
  st.bytes += (unsigned)rows * 128u;
}

// ---- 32x32 tile product over a staged panel ----------------------------------------------------------
// 256 threads = 16 k-groups x (4 x 4) threads, each thread an 8x8 register micro-tile: 16 LDS.128 per
// 256 FFMA.  (The first version used 4 k-groups x 4x4 micro-tiles = 8 LDS.128 per 64 FFMA; every LDS.128
// costs 4 shared-memory phases whatever the broadcast pattern, so that shape was shared-memory-bandwidth
// bound at <= 50 % of the FFMA rate.)  Rows/cols are interleaved (r = ty + 4 i) for k-contiguous panels so
// a quarter-warp's 16-byte reads fall in distinct banks, contiguous (r = 8 ty + i) for dense [k][32] panels
// (no padding needed there: the 8 lanes of one LDS.128 phase read at most 4 distinct 32-byte spans of one row).
template <bool A_KC, bool B_KC>
__device__ __forceinline__ void tile_mma(const float* As, const float* Bs, int kp, float (&acc)[8][8], float* rs) {
  const int tid = threadIdx.x, grp = tid >> 4, t = tid & 15, tx = t & 3, ty = t >> 2;
  const int a_stride = kp + 4, b_stride = kp + 4;
  for (int k = grp * 4; k < kp; k += 4 * KG) {
    float a[8][4], b[8][4];
    if (A_KC) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(&As[(ty + 4 * i) * a_stride + k]);
        a[i][0] = v.x; a[i][1] = v.y; a[i][2] = v.z; a[i][3] = v.w;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v0 = *reinterpret_cast<const float4*>(&As[(k + q) * 32 + ty * 8]);
        const float4 v1 = *reinterpret_cast<const float4*>(&As[(k + q) * 32 + ty * 8 + 4]);
        a[0][q] = v0.x; a[1][q] = v0.y; a[2][q] = v0.z; a[3][q] = v0.w;
        a[4][q] = v1.x; a[5][q] = v1.y; a[6][q] = v1.z; a[7][q] = v1.w;
      }
    }
    if (B_KC) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 v = *reinterpret_cast<const float4*>(&Bs[(tx + 4 * j) * b_stride + k]);
        b[j][0] = v.x; b[j][1] = v.y; b[j][2] = v.z; b[j][3] = v.w;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v0 = *reinterpret_cast<const float4*>(&Bs[(k + q) * 32 + tx * 8]);
        const float4 v1 = *reinterpret_cast<const float4*>(&Bs[(k + q) * 32 + tx * 8 + 4]);
        b[0][q] = v0.x; b[1][q] = v0.y; b[2][q] = v0.z; b[3][q] = v0.w;
        b[4][q] = v1.x; b[5][q] = v1.y; b[6][q] = v1.z; b[7][q] = v1.w;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i][q], b[j][q], acc[i][j]);
    if (rs) {
#pragma unroll
      for (int i = 0; i < 8; ++i) rs[i] += (a[i][0] + a[i][1]) + (a[i][2] + a[i][3]);
    }
  }
}

template <bool A_KC>
__device__ __forceinline__ int tile_row(int ty, int i) { return A_KC ? (ty + 4 * i) : (ty * 8 + i); }

// fold the 16 k-groups in a fixed order; thread gets outputs e = tid + r*256 -> (m = e>>5, n = e&31).
// The caller has synchronised the CTA since the last read of the memory behind `red` (RED_FLOATS), and synchronises
// it again before anyone writes there (no trailing barrier here: P1's next writer is already behind the ticket's).
// Row i of thread (ty, tx) always goes to row slot ty + 4 i of its group's 32 x 36 block and its 8 elements to column
// slots 8 tx .. 8 tx + 7, whatever tile row / columns they stand for: two 16-byte stores per row, and the 8 lanes of a
// quarter-warp phase (tx = 0..3, two ty) cover 32 distinct banks (group blocks are 16 banks apart).  The reader maps
// its output (m, n) back through the panels' row / column orders; a warp reads one row slot, 32 distinct banks.
constexpr int RED_GS = 32 * 36 + 16;
template <bool KC>
__device__ __forceinline__ int red_row(int m) { return KC ? m : ((m >> 3) + 4 * (m & 7)); }
template <bool KC>
__device__ __forceinline__ int red_col(int n) { return KC ? (8 * (n & 3) + (n >> 2)) : n; }
template <bool A_KC, bool B_KC>
__device__ __forceinline__ void tile_reduce(const float (&acc)[8][8], float* red, float (&outv)[4]) {
  const int tid = threadIdx.x, grp = tid >> 4, t = tid & 15, tx = t & 3, ty = t >> 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float4* p = reinterpret_cast<float4*>(&red[grp * RED_GS + (ty + 4 * i) * 36 + 8 * tx]);
    p[0] = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    p[1] = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int e = tid + r * NT, m = e >> 5, n = e & 31;
    const int off = red_row<A_KC>(m) * 36 + red_col<B_KC>(n);
    float g_[KG];
#pragma unroll
    for (int g = 0; g < KG; ++g) g_[g] = red[g * RED_GS + off];
    float v = 0.f;
#pragma unroll
    for (int g = 0; g < KG; ++g) v += g_[g];
    outv[r] = v;
  }
}

// fixed-order block sum of one float (all threads call; every thread gets the result)
__device__ __forceinline__ float block_sum(float v, float* scratch /*[8]*/) {
  v = jb_warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) t += scratch[w];
  return t;
}

// one level of the head-output butterfly: lanes with bit N set keep the upper half of values [0, 2N), the others the
// lower half, and each adds the half its partner sent.  One template instance per level so that every index into h is a
// compile-time constant: a loop over the levels left h in local memory (a load-shuffle-store round trip per value).
__device__ __forceinline__ float butterfly_pair(float lo, float hi, bool up, int N) {
  return (up ? hi : lo) + __shfl_xor_sync(0xffffffffu, up ? lo : hi, N);
}
template <int N, int S>
__device__ __forceinline__ void butterfly_level(float (&h)[S], int lane) {
  static_assert(2 * N <= S, "butterfly level wider than its values");
  const bool up = (lane & N) != 0;
#pragma unroll
  for (int q = 0; q < N; ++q) h[q] = butterfly_pair(h[q], h[q + N], up, N);
}

// d (loss) / d (h2 pre-activation) for 4 adjacent columns of one row: (dout[row] . Wh[:, c..c+3]) * relu'(h2).
// MO >= nout bounds the head outputs: dout and wr are zero beyond nout, and each term left out would be fmaf(0, 0, t),
// which returns t (the sum of +0 and a zero t is +0 where t = -0; the relu mask, the tile products and the squares of
// the norm do not tell the two zeros apart).
template <int MO>
__device__ __forceinline__ float4 dh2_quad(const float* drow, const float4 (&wr)[MAXO], float4 hv) {
  static_assert(MO >= 1 && MO <= MAXO, "head output bound");
  const float4 d0 = *reinterpret_cast<const float4*>(drow);
  const float4 d1 = *reinterpret_cast<const float4*>(drow + 4);
  const float d[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
  float4 t = make_float4(d[0] * wr[0].x, d[0] * wr[0].y, d[0] * wr[0].z, d[0] * wr[0].w);
#pragma unroll
  for (int o = 1; o < MO; ++o) {
    t.x = fmaf(d[o], wr[o].x, t.x); t.y = fmaf(d[o], wr[o].y, t.y); t.z = fmaf(d[o], wr[o].z, t.z); t.w = fmaf(d[o], wr[o].w, t.w);
  }
  return make_float4(hv.x > 0.f ? t.x : 0.f, hv.y > 0.f ? t.y : 0.f, hv.z > 0.f ? t.z : 0.f, hv.w > 0.f ? t.w : 0.f);
}

// ---- tensor-core phases (TC instantiation): 3xTF32 wgmma products, building blocks in csrc/wgmma.cuh ----------------
using jbwg::tile_off;
__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(mbar), "r"(count) : "memory");
}
// Bounded: a tensor-core pipeline bug must fail the launch (trap -> CUDA error on the host), never hang the GPU.  The
// bound is counted in SM clock cycles (clock64 is a register read; %globaltimer costs microseconds per read, which made
// every wait that missed its first try a multi-microsecond stall).
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
  unsigned done = 0;
  const long long t0 = clock64();
  for (;;) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n" : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
    if (done) return;
    if (clock64() - t0 > (1ll << 32)) asm volatile("trap;\n");      // ~2 s
  }
}
__device__ __forceinline__ void mbar_expect_tx(unsigned mbar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
// the low part of the 3xTF32 split: x - trunc_tf32(x) (the tensor core truncates the raw fp32 word), rounded to tf32
__device__ __forceinline__ float tf32_lo(float x) {
  const float r = x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  unsigned o;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(o) : "f"(r));
  return __uint_as_float(o);
}
constexpr int TC_A_BYTES = 2 * 128 * 128;        // one A chunk: hi | lo, each [128 rows][32 k] fp32 = 16 KB
constexpr int TC_B_BYTES = 2 * 32 * 128;         // one B chunk: hi | lo, each [32 rows][32 k] fp32 = 4 KB
constexpr int TC_NA = 3, TC_NB = 5;              // ring depths: A chunks are generated, B chunks stream in 4 ahead (+ 8 KB: x tile)
constexpr int TC_BAR_WORD = 1664;                // s_small word offset of the tensor-core mbarriers (8 x 8 bytes)
constexpr int TC_BAR_JB = TC_NB;                 // [0..4] forward B chunk landed, [5..7] dh1 jobs' W2^T chunk landed
constexpr int TC_NBAR = TC_NB + TC_NA;
constexpr int TC_LD = 36;                        // row stride (floats) of the [128][32] accumulator image the epilogues read

// timing trace (debug; JB_FUSED_SKIP bit 8): clock64 at fixed points of the LAST step, per CTA, 32 slots
__device__ long long g_trace[256 * 48];
#define TR(i) do { if (trace && tid == 0) g_trace[cta * 48 + (i)] = clock64(); } while (0)

struct HeadTab { const float* w[MAXO]; const float* b[MAXO]; float* gw[MAXO]; float* gb[MAXO]; };

// TC: tensor-core phases (B % 128 == 0, H % 128 == 0); NA / ND: compile-time bounds on the action count / the input
// dimension (loop bounds of the row maths / of the operand generators: a D = 4 net must not pay for 16 predicated slots)
template <bool TC, int NA, int ND>
__global__ void __launch_bounds__(NT, 1) ppo_epoch_kernel(Args a, int dsm_floats, int flags /* debug: bit 8 = trace */) {
  extern __shared__ __align__(16) float smem[];
  float* s_small = smem;                       // SMALL_FLOATS
  float* dsm = smem + SMALL_FLOATS;            // d loss/d head-outputs of the whole minibatch [B][MAXO] (P1: rollout values)
  float* R0 = dsm + dsm_floats;                // RED_FLOATS: A panels of P1 / JB, split-K fold area, job scratch
  float* R1 = R0 + RED_FLOATS;                 // RED_FLOATS: B panels
  float* R2 = R1 + RED_FLOATS;                 // R2_FLOATS:  A panel of JA / JC; W1 during P1
  float* PS = R2 + R2_FLOATS;                  // PS_FLOATS:  head weight rows, b2, b1 of the current step
  float* xs = s_small;                         // [MAXD][32] state rows of the current tile, transposed (zero padded)
  float* scr = s_small + 768;                  // reduction scratch [128]
  int* sidx = reinterpret_cast<int*>(s_small + 1024);   // [32] gathered rollout row ids of the P1 tile
  Stager st;
  st.init(s_small + 1056);                     // 8-byte mbarrier: panels
  Stager stp;
  stp.init(s_small + 1058);                    // 8-byte mbarrier: parameter stash
  float* dvs = s_small + 1088;                 // [MAX_B] second candidate value-head gradient of every row (P3); norm partials (P5)
  float* hb = s_small + 1600;                  // [MAXO] head biases
  // tensor-core phases (TC instantiation): operand rings inside R0..R1 (1 KB aligned), TC_NBAR mbarriers for the bulk
  // copies; each warpgroup keeps its 64 x 32 accumulator in registers (csrc/wgmma.cuh)
  unsigned tc_base = 0;
  unsigned long long tc_g = 0;                 // chunks issued so far by this CTA: ring positions and mbarrier phases
  unsigned long long jb_g = 0;                 // same for the tensor-core dh1 jobs
  unsigned long long ja_g = 0;                 // ... and the dW2 jobs
  const unsigned tc_bar = smem_u32(s_small + TC_BAR_WORD);
  float* tcp = nullptr;                        // generic pointer to the ring base (epilogue scratch)
  float* tcs = nullptr;                        // [128][TC_LD] accumulator image for the epilogues (A ring slot 1)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = tid >> 7;
  const unsigned int nctas = gridDim.x;
  const int cta = blockIdx.x;
  const int B = a.B, D = a.D, H = a.H, A = a.A, nout = a.nout;
  const int npol = a.continuous ? 2 * A : A;
  constexpr int NO = 2 * NA + 1 < MAXO ? 2 * NA + 1 : MAXO;   // >= nout = npol + 1 (the host picks NA >= A)
  const int nq = (nout + 3) >> 2;              // float4 quads of head outputs per row
  const float invB = 1.0f / (float)B;
  const jbppo::HP hp{a.eps_clip, a.vf_coef, a.ent_coef};
  unsigned int epoch = 0;
  const long long step0 = *a.step, cursor0 = *a.cursor;
  const float lr = *a.lr;

  if (TC) {
    tc_base = (smem_u32(R0) + 1023u) & ~1023u;
    tcp = R0 + ((tc_base - smem_u32(R0)) >> 2);
    tcs = tcp + TC_A_BYTES / 4;
    if (tid == 0) {
      for (int i = 0; i < TC_NBAR; ++i) mbar_init(tc_bar + 8u * i, 1);
      asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
  }
  HeadTab& ht = *reinterpret_cast<HeadTab*>(s_small + 896);   // 32 pointers: shared memory, not 64 live registers
  if (tid == 0) {
    int o = 0;
    for (int g = 0; g < 3; ++g)
      for (int q = 0; q < a.nh[g]; ++q, ++o) {
        ht.w[o] = a.Wh[g] + (size_t)q * H; ht.b[o] = a.bh[g] + q; ht.gw[o] = a.gWh[g] + (size_t)q * H; ht.gb[o] = a.gbh[g] + q;
      }
    for (; o < MAXO; ++o) { ht.w[o] = a.Wh[0]; ht.b[o] = a.bh[0]; ht.gw[o] = a.gWh[0]; ht.gb[o] = a.gbh[0]; }
  }
  __syncthreads();

  const int MT = B / 32, NTL = H / 32, NP = (NTL + 1) >> 1;
  const int nJ1 = TC ? (B >> 7) * NTL : MT * NTL;   // P1 tiles: 128 x 32 on the tensor cores, else 32 x 32 FFMA tiles
  const int nJB = TC ? (H >> 7) * MT : MT * NTL;   // dh1 tiles: TC 128 (hidden units) x 32 (rows), else 32 x 32 like P1
  const int nJA = TC ? (H >> 7) * NTL : NTL * NP;   // dW2: TC 128 (k) x 32 (n) tiles of dW2^T, else pairs of 32 x 32 tiles
  const int nJC = NTL;               // head weight-gradient column jobs
  const int nJD = NTL;               // dW1 / db1 folds
  const int nJ3 = nJB + nJA + nJC + nJD;
  const bool single = B <= JA_ROWS;  // one panel covers the minibatch: JA pairs share their generated panel

  // Adam: static slice of the flat buffers; bias-correction powers advance by one multiply per step
  const long long per = (a.P4 + nctas - 1) / nctas;
  const long long lo = (long long)cta * per, hi = min(a.P4, lo + per);
  float4* p4 = reinterpret_cast<float4*>(a.flat);
  const float4* g4 = reinterpret_cast<const float4*>(a.grad);
  float4* m4 = reinterpret_cast<float4*>(a.am);
  float4* v4 = reinterpret_cast<float4*>(a.av);
  double pw1 = pow((double)a.beta1, (double)(step0 + 1)), pw2 = pow((double)a.beta2, (double)(step0 + 1));
  // W2t: tiled shadow of W2 ([H/32][H][32]: W2t[kt][n][c] = W2[n][32 kt + c]) so that the B panel of a JB job is
  // one contiguous 64 KB block; the owner of a float4 of W2 in the Adam phase also writes its shadow
  const long long w2_lo = (long long)(a.W2 - a.flat) >> 2, w2_hi = w2_lo + (long long)H * H / 4;
  auto shadow = [&](long long i, float4 v) {
    if (i >= w2_lo && i < w2_hi) {
      const int e = (int)(i - w2_lo) * 4, n = e / H, k = e - n * H;
      *reinterpret_cast<float4*>(&a.W2t[((size_t)(k >> 5) * H + n) * 32 + (k & 31)]) = v;
      if (TC) {
        // wgmma-ready images of W2 (hi | lo of the 3xTF32 split): tile (n / 32, k / 32) = [32 rows][32 k] in the swizzled
        // K-major layout, so that a B chunk of the forward phase is ONE 4 KB bulk copy per image
        float* img = a.W2img + ((size_t)(n >> 5) * (H >> 5) + (k >> 5)) * 1024 + (tile_off(n & 31, (k & 31) >> 2) >> 2);
        *reinterpret_cast<float4*>(img) = v;
        *reinterpret_cast<float4*>(img + (size_t)H * H) = make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w));
        // ... and of W2^T for the dh1 jobs: tile (k / 128, n / 32) = [128 rows k][32 columns n]
        const float vv4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int kk = k + q;
          float* t = a.W2Timg + ((size_t)(kk >> 7) * (H >> 5) + (n >> 5)) * 4096 + (tile_off(kk & 127, (n & 31) >> 2) >> 2) + (n & 3);
          t[0] = vv4[q];
          t[(size_t)H * H] = tf32_lo(vv4[q]);
        }
      }
    }
  };
  for (long long i = lo + tid; i < hi; i += NT) shadow(i, p4[i]);   // published by the first grid barrier
  const float one_m_b1 = 1.f - a.beta1, one_m_b2 = 1.f - a.beta2;

  // first-panel cp.async of a backward job (JD has none); b_in_flight: a JB job's W2t panel was issued before bar1
  auto issue_stage = [&](int job, bool b_in_flight) {
    if (job < nJB) {
      if (TC) return;                          // tensor-core dh1 jobs run their own operand rings
      const int mt = job / NTL, kt = job - mt * NTL;
      stage_kc(st, R0, a.h2, H, mt * 32, 0, H);
      if (!b_in_flight) stage_block(st, R1, a.W2t + (size_t)kt * H * 32, H);
    } else if (job < nJB + nJA) {
      if (TC) return;                          // tensor-core dW2 jobs generate both operands
      const int j = job - nJB, nt = j / NP, kt0 = 2 * (j - nt * NP), kp = min(JA_ROWS, B);
      stage_block(st, R2, a.h2t + (size_t)nt * B * 32, kp);
      stage_block(st, R1, a.h1 + (size_t)kt0 * B * 32, kp);
      if (single && kt0 + 1 < NTL) stage_block(st, R1 + R2_FLOATS, a.h1 + (size_t)(kt0 + 1) * B * 32, kp);
    } else if (job < nJB + nJA + nJC) {
      stage_block(st, R2, a.h2t + (size_t)(job - nJB - nJA) * B * 32, min(JA_ROWS, B));
    }
    st.commit();
  };
  // may the panels of `job` be fetched while the previous job still folds in R0?
  auto prefetchable = [&](int job) { return job < nJ3 && job >= nJB && (single || job >= nJB + nJA); };

  // ---- loss row maths, run for the rows of a P1 row tile by the CTA that finishes the tile's LAST column tile (it draws
  // the last ticket of a.barrier[CTR_ROW + mt]; nobody waits on the tickets).  The rollout values of a row (adv, ret, v_old,
  // log_prob_old, action: every row is visited once per epoch, so these are cold misses) are fetched at the start of the
  // P1 tile by the thread that will need them, into dsm [6][RW] (dsm is free until bar1); the results go to global tables
  // that bar1 publishes.
  const int RW = TC ? 128 : 32;                        // rows of a P1 tile
  auto gather_row = [&](int i, int r) {                // tile row i = rollout row r
    cp_async4(dsm + i, a.adv + r); cp_async4(dsm + RW + i, a.ret + r); cp_async4(dsm + 2 * RW + i, a.vold + r);
    if (!a.continuous) { cp_async4(dsm + 3 * RW + i, a.logp_old + r); cp_async4(dsm + 4 * RW + i, (const int32_t*)a.action + r); }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    dsm[5 * RW + i] = __int_as_float(r);
  };
  auto row_maths = [&](int b, int i) {
    const float g_adv = dsm[i], g_ret = dsm[RW + i], g_vold = dsm[2 * RW + i], g_lpo = dsm[3 * RW + i];
    const int g_act = __float_as_int(dsm[4 * RW + i]), r = __float_as_int(dsm[5 * RW + i]);
    float ov[2 * jbppo::MAX_A + 1];                     // row() indexes up to 2*MAX_A statically
#pragma unroll
    for (int o = 0; o < 2 * jbppo::MAX_A + 1; ++o) ov[o] = 0.f;
#pragma unroll
    for (int o = 0; o < MAXO; ++o) if (o < nout) ov[o] = hb[o];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (q < nq) {                                    // 16 independent loads in flight, folded in tile order
        float4 v[PK / 32];
#pragma unroll
        for (int nt = 0; nt < PK / 32; ++nt)      // clamped, not predicated: all 16 loads go out back to back
          v[nt] = ldcg4(a.headp + (((size_t)min(nt, NTL - 1) * 2 + q) * B + b) * 4);
#pragma unroll
        for (int nt = 0; nt < PK / 32; ++nt) {
          if (nt < NTL) { ov[q * 4] += v[nt].x; ov[q * 4 + 1] += v[nt].y; ov[q * 4 + 2] += v[nt].z; ov[q * 4 + 3] += v[nt].w; }
        }
      }
    }
    jbppo::RowOut ro;
    if (a.continuous)
      jbppo::row<true, NA>(ov, A, 0, (const float*)a.action + (size_t)r * A, g_adv, g_ret, g_vold,
                           a.logp_old + (size_t)r * A, hp, invB, ro);
    else
      jbppo::row<false, NA>(ov, A, g_act, nullptr, g_adv, g_ret, g_vold, &g_lpo, hp, invB, ro);
    // d loss / d head outputs; the value head's slot holds the critic_loss1 candidate, resolved after bar1
    float d[MAXO];
#pragma unroll
    for (int o = 0; o < MAXO; ++o) d[o] = o < npol ? ro.dpol[o] : (o == npol ? ro.dv1 : 0.f);
    static_assert(MAXO == 8, "dout rows are two float4 ([B][8] in ppo_fused.py)");
    float4* dst = reinterpret_cast<float4*>(a.dout + (size_t)b * MAXO);
    dst[0] = make_float4(d[0], d[1], d[2], d[3]);
    dst[1] = make_float4(d[4], d[5], d[6], d[7]);
    a.dv2[b] = ro.dv2;
    // the differences, not their squares: after bar1 the critic sums are `p += d * d`, one FMA per row (a stored square
    // would be rounded once more)
    float* st_ = a.rowst + b;
    st_[0] = ro.d1; st_[B] = ro.d2; st_[2 * B] = ro.surr_min; st_[3 * B] = ro.ent; st_[4 * B] = ro.ratio; st_[5 * B] = ro.pmin;
  };
  int* tkt = reinterpret_cast<int*>(s_small + 1060);  // "this CTA drew the last ticket"
  // state rows of this CTA's first P1 tile of step 0 (later steps: gathered under the Adam phase)
  bool xs_ready = false;
  float xpre[ND];                                // TC: this thread's state row (row tid & 127 of the CTA's first tile)
  int xpre_idx = 0;
#pragma unroll
  for (int i = 0; i < ND; ++i) xpre[i] = 0.f;
  if (TC && cta < nJ1) {
    xpre_idx = a.perm[cursor0 * (long long)B + (cta / NTL) * 128 + (tid & 127)];
#pragma unroll
    for (int i = 0; i < ND; ++i) if (i < D) xpre[i] = a.state[(size_t)xpre_idx * D + i];
    xs_ready = true;
  }
  if (!TC && cta < nJ1) {
    if (tid < 32) sidx[tid] = a.perm[cursor0 * (long long)B + (cta / NTL) * 32 + tid];
    __syncthreads();
    for (int e = tid; e < 32 * MAXD; e += NT) { const int r = e >> 4, i = e & 15; xs[i * 32 + r] = i < D ? a.state[(size_t)sidx[r] * D + i] : 0.f; }
    xs_ready = true;
  }
  __syncthreads();

  if (TC) grid_bar(a.barrier, epoch, nctas);     // the W2 images built above are read by the FIRST forward phase

  for (int s = 0; s < a.n_steps; ++s) {
    const bool trace = (flags & 256) && s == a.n_steps - 1;
    TR(0);
    __syncthreads();                               // (step 0: the prologue; later steps: a no-op after the barrier)
    // =========================== P1: h2 = relu(relu(x W1^T + b1) W2^T + b2), partial head outputs ========
    // parameter stash: ONE bulk request per tensor per CTA, issued from different warps.  (Per-thread loads of
    // W1 / b1 / b2 / head rows had every warp of every CTA hit the same few KB right after the barrier: > 500 K
    // sector requests queued on ~100 L2 lines, microseconds before the first value arrived.)
    stp.bytes = (unsigned)(H * D + (2 + nout) * H) * 4u;
    stp.commit();                                  // thread 0 arrives with the byte count before anything else
    if (tid == 32) stp.copy(R2, a.W1, (unsigned)(H * D) * 4u);
    if (tid == 64) { stp.copy(PS + (MAXO + 1) * PK, a.b1, (unsigned)H * 4u); stp.copy(PS + MAXO * PK, a.b2, (unsigned)H * 4u); }
    if (tid >= 96 && tid < 96 + nout) stp.copy(PS + (tid - 96) * PK, ht.w[tid - 96], (unsigned)H * 4u);
    if (tid >= 128 && tid < 128 + nout) hb[tid - 128] = ldcg(ht.b[tid - 128]);
    if (!TC && cta < nJ1) { stage_kc(st, R1, a.W2, H, (cta % NTL) * 32, 0, H); st.commit(); }
    TR(28);
    stp.wait();
    TR(29);
    bool w2t_pre = false;                          // B panel of the first JB job already in flight (FFMA engine)
    // one ticket per finished P1 tile of row tile mt: the CTA that draws the last one runs the row maths of the tile's rows
    auto row_ticket = [&](int mt, bool mine, int b, int i) {
      if (mine) asm volatile("cp.async.wait_all;\n" ::: "memory");   // the tile's rollout values (landed long ago)
      __syncthreads();                             // every thread's headp stores happen-before thread 0's release
      if (tid == 0) {
        unsigned int old;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;\n" : "=r"(old) : "l"(a.barrier + CTR_ROW + mt) : "memory");
        *tkt = old + 1u == (unsigned int)NTL * (unsigned int)(s + 1);
      }
      __syncthreads();
      TR(36);
      if (*tkt) {
        if (mine) row_maths(b, i);
        TR(37);
      }
    };
    if constexpr (TC) {
      // ---- tensor-core forward: one 128 (minibatch rows) x 32 (hidden units) tile per job, K = H in chunks of 32.
      // A chunk = h1[128 rows][32 k] = relu(x W1^T + b1), GENERATED straight into the swizzled K-major layout (hi | lo of
      // the 3xTF32 split) by all threads; B chunk = hi | lo image of W2[n0..n0+32][32 k] (kept current by the Adam phase),
      // one 8 KB pair of bulk copies four chunks ahead; each warpgroup issues 4 x 3 wgmma (m64n32k8, tf32) per chunk for its
      // 64 rows and leaves them in flight while the next chunk is generated into another A slot.
      const int NKC = H >> 5;
      for (int job = cta; job < nJ1; job += (int)nctas) {
        const int mt = job / NTL, nt = job - mt * NTL, m0 = mt * 128, n0 = nt * 32;
        const int r = tid & 127, half = tid >> 7;
        auto issue_b = [&](int kc, unsigned long long g) {
          const unsigned slot = (unsigned)(g % TC_NB);
          const unsigned bar = tc_bar + 8u * slot, dst = tc_base + TC_NA * TC_A_BYTES + slot * TC_B_BYTES;
          mbar_expect_tx(bar, TC_B_BYTES);
          const float* src = a.W2img + ((size_t)nt * NKC + kc) * 1024;
          bulk_g2s(dst, src, 4096u, bar);
          bulk_g2s(dst + 4096u, src + (size_t)H * H, 4096u, bar);
        };
        if (tid == 0)
          for (int kc = 0; kc < min(TC_NB - 1, NKC); ++kc) issue_b(kc, tc_g + kc);
        float xr[ND];
        int xidx;
        if (job == cta && xs_ready) {
          xidx = xpre_idx;
#pragma unroll
          for (int i = 0; i < ND; ++i) xr[i] = xpre[i];
        } else {
          xidx = a.perm[(cursor0 + s) * (long long)B + m0 + r];
#pragma unroll
          for (int i = 0; i < ND; ++i) xr[i] = i < D ? a.state[(size_t)xidx * D + i] : 0.f;
        }
        if (nt == 0 && half == 0) {
          a.cur_idx[m0 + r] = xidx;
          for (int i = 0; i < D; ++i) a.xg[(size_t)(m0 + r) * D + i] = xr[i];
        }
        if (half == 0) gather_row(r, xidx);
        // the tile's 128 input rows, transposed [ND][128], in the spare 8 KB behind the operand rings: the generator
        // below reads them as broadcast float4 (4 rows of one input feature)
        float* xt = tcp + ((TC_NA * TC_A_BYTES + TC_NB * TC_B_BYTES) >> 2);
        __syncthreads();                                          // previous tile's generators are done with xt
        if (half == 0) {
#pragma unroll
          for (int i = 0; i < ND; ++i) xt[i * 128 + r] = xr[i];
        }
        __syncthreads();
        const float* W1s = R2;
        const float* b1s = PS + (MAXO + 1) * PK;
        float acc[16];
        TR(1);
        for (int kc = 0; kc < NKC; ++kc) {
          const unsigned long long g = tc_g + kc;
          const unsigned abuf = tc_base + (unsigned)(g % TC_NA) * TC_A_BYTES;   // chunk g - 3's slot: retired (wait below)
          // generator: lane = hidden unit 32 kc + lane (its W1 row in registers), warp = rows 16 warp .. + 15
          const int k = kc * 32 + lane;
          float w1k[ND];
#pragma unroll
          for (int i = 0; i < ND; ++i) w1k[i] = i < D ? W1s[k * D + i] : 0.f;
          const float b1k = b1s[k];
          float hv[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) hv[j] = 0.f;
#pragma unroll
          for (int i = 0; i < ND; ++i) {
            if (i < D) {
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const float4 x4 = *reinterpret_cast<const float4*>(&xt[i * 128 + warp * 16 + 4 * c]);
                hv[4 * c] = fmaf(x4.x, w1k[i], hv[4 * c]); hv[4 * c + 1] = fmaf(x4.y, w1k[i], hv[4 * c + 1]);
                hv[4 * c + 2] = fmaf(x4.z, w1k[i], hv[4 * c + 2]); hv[4 * c + 3] = fmaf(x4.w, w1k[i], hv[4 * c + 3]);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int row = warp * 16 + j;
            const float hi = fmaxf(hv[j] + b1k, 0.f);
            const unsigned off = tile_off(row, lane >> 2) + ((unsigned)(lane & 3) << 2);
            asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(abuf + off), "f"(hi) : "memory");
            asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(abuf + 16384u + off), "f"(tf32_lo(hi)) : "memory");
            if (nt == 0) a.h1[((size_t)kc * B + m0 + row) * 32 + lane] = hi;                  // tiled [H/32][B][32]
          }
          jbwg::wait<0>();                                              // chunk g - 1's products of this warpgroup retired
          jbwg::fence_acc(acc);
          asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // generic-proxy stores -> async proxy (wgmma reads)
          __syncthreads();                                              // ... and those of the other warpgroup
          const unsigned slot = (unsigned)(g % TC_NB);
          if (tid == 0 && kc + TC_NB - 1 < NKC) issue_b(kc + TC_NB - 1, g + TC_NB - 1);   // chunk kc + 4 where chunk kc - 1 lived
          mbar_wait(tc_bar + 8u * slot, (unsigned)((g / TC_NB) & 1));   // B chunk landed
          const unsigned bbuf = tc_base + TC_NA * TC_A_BYTES + slot * TC_B_BYTES, aw = abuf + (unsigned)wg * 8192u;
          jbwg::fence();
          jbwg::mma3_n32(acc, aw, aw + 16384u, bbuf, bbuf + 4096u, kc == 0);
          jbwg::commit();
        }
        TR(3);
        // ---- epilogue: accumulator image in shared memory, then thread = one row of 16 columns (warp w: rows 32 (w & 3)..,
        // columns 16 (w >> 2)..): bias + relu, h2 in both layouts, partial head outputs of the tile's 32 columns
        jbwg::wait<0>();
        jbwg::fence_acc(acc);
        __syncthreads();                                          // both warpgroups' products retired: tcs overlays A slot 1
        jbwg::store_acc_n32(acc, tcs, TC_LD);
        __syncthreads();
        {
          const int q = warp & 3, cb = (warp >> 2) * 16, row = m0 + q * 32 + lane;
          float rr[16];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 t = *reinterpret_cast<const float4*>(&tcs[(q * 32 + lane) * TC_LD + cb + 4 * c]);
            rr[4 * c] = t.x; rr[4 * c + 1] = t.y; rr[4 * c + 2] = t.z; rr[4 * c + 3] = t.w;
          }
          float v[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] = fmaxf(rr[i] + PS[MAXO * PK + n0 + cb + i], 0.f);
          float4* o2 = reinterpret_cast<float4*>(a.h2 + (size_t)row * H + n0 + cb);
          float4* o2t = reinterpret_cast<float4*>(a.h2t + ((size_t)nt * B + row) * 32 + cb);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 t = make_float4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
            o2[c] = t; o2t[c] = t;
          }
          float ph[MAXO];
#pragma unroll
          for (int o = 0; o < MAXO; ++o) {
            float t = 0.f;
            if (o < nout) {
#pragma unroll
              for (int i = 0; i < 16; ++i) t = fmaf(v[i], PS[o * PK + n0 + cb + i], t);
            }
            ph[o] = t;
          }
          float* sc = tcp + (q * 32 + lane) * MAXO;              // ring slot 0: every MMA that read it has retired
          if (warp >= 4) {
            *reinterpret_cast<float4*>(sc) = make_float4(ph[0], ph[1], ph[2], ph[3]);
            *reinterpret_cast<float4*>(sc + 4) = make_float4(ph[4], ph[5], ph[6], ph[7]);
          }
          __syncthreads();
          if (warp < 4) {
            const float4 u0 = *reinterpret_cast<const float4*>(sc), u1 = *reinterpret_cast<const float4*>(sc + 4);
            *reinterpret_cast<float4*>(a.headp + (((size_t)nt * 2 + 0) * B + row) * 4) = make_float4(ph[0] + u0.x, ph[1] + u0.y, ph[2] + u0.z, ph[3] + u0.w);
            if (nq > 1)
              *reinterpret_cast<float4*>(a.headp + (((size_t)nt * 2 + 1) * B + row) * 4) = make_float4(ph[4] + u1.x, ph[5] + u1.y, ph[6] + u1.z, ph[7] + u1.w);
          }
          __syncthreads();
        }
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // scratch reads above before later bulk copies / wgmma
        tc_g += (unsigned long long)NKC;
        TR(4);
        row_ticket(mt, half == 0, m0 + r, r);
      }
    } else
    for (int job = cta; job < nJ1; job += (int)nctas) {
      const int mt = job / NTL, nt = job - mt * NTL;
      const int m0 = mt * 32, n0 = nt * 32;
      if (job != cta) {
        __syncthreads();
        stage_kc(st, R1, a.W2, H, n0, 0, H);
        st.commit();
      }
      if (!(job == cta && xs_ready)) {
        if (tid < 32) sidx[tid] = a.perm[(cursor0 + s) * (long long)B + m0 + tid];
        __syncthreads();
        for (int e = tid; e < 32 * MAXD; e += NT) { const int r = e >> 4, i = e & 15; xs[i * 32 + r] = i < D ? a.state[(size_t)sidx[r] * D + i] : 0.f; }
        __syncthreads();
      }
      if (tid < 32) gather_row(tid, sidx[tid]);
      if (nt == 0) {
        if (tid < 32) a.cur_idx[m0 + tid] = sidx[tid];
        for (int e = tid; e < 32 * D; e += NT) { const int r = e / D, i = e - r * D; a.xg[(size_t)(m0 + r) * D + i] = xs[i * 32 + r]; }
      }
      {
        // h1 panel: warp = (row half, block of 128 hidden units); thread = units 128 kw + 32 j + lane, j < 4, x 16 rows.
        // One compact loop body per unit (the fully unrolled form was ~2000 instructions executed once per step:
        // instruction-fetch bound).
        const int rh = warp >> 2, kbase = (warp & 3) * 128 + lane;
        const float* W1s = R2;
        const float* b1s = PS + (MAXO + 1) * PK;
        const float* xcol = xs + rh * 16;          // x[i][rh*16 .. +16): four LDS.128 per input feature
#pragma unroll 1
        for (int j = 0; j < 4; ++j) {
          const int k = kbase + 32 * j;
          if (k >= H) break;
          float h[16];
#pragma unroll
          for (int r = 0; r < 16; ++r) h[r] = 0.f;
          auto feature = [&](int i) {
            const float w = W1s[k * D + i];
#pragma unroll
            for (int r4 = 0; r4 < 4; ++r4) {
              const float4 x = *reinterpret_cast<const float4*>(&xcol[i * 32 + r4 * 4]);
              h[r4 * 4] = fmaf(x.x, w, h[r4 * 4]); h[r4 * 4 + 1] = fmaf(x.y, w, h[r4 * 4 + 1]);
              h[r4 * 4 + 2] = fmaf(x.z, w, h[r4 * 4 + 2]); h[r4 * 4 + 3] = fmaf(x.w, w, h[r4 * 4 + 3]);
            }
          };
          if constexpr (ND <= 4) {                 // D <= 4 (CartPole): the input features unrolled, their 16 shared-memory loads in
#pragma unroll                                     // flight together (the rolled loop exposed one load latency per feature)
            for (int i = 0; i < ND; ++i) if (i < D) feature(i);
          } else {
#pragma unroll 1
            for (int i = 0; i < D; ++i) feature(i);
          }
          const float bb = b1s[k];
          float* ps = R0 + rh * 16 * (H + 4) + k;
#pragma unroll
          for (int r = 0; r < 16; ++r) { h[r] = fmaxf(h[r] + bb, 0.f); ps[r * (H + 4)] = h[r]; }
          if (nt == 0) {
            float* pgl = a.h1 + ((size_t)(k >> 5) * B + m0 + rh * 16) * 32 + (k & 31);   // tiled [H/32][B][32]
#pragma unroll
            for (int r = 0; r < 16; ++r) pgl[r * 32] = h[r];
          }
        }
      }
      float whr[MAXO];
#pragma unroll
      for (int o = 0; o < MAXO; ++o) whr[o] = o < nout ? PS[o * PK + n0 + lane] : 0.f;
      const float b2v = PS[MAXO * PK + n0 + lane];
      TR(1);
      st.wait();
      __syncthreads();
      TR(2);
      float acc[8][8] = {};
      tile_mma<true, true>(R0, R1, H, acc, nullptr);
      __syncthreads();
      TR(3);
      if (s > 0 && job + (int)nctas >= nJ1 && cta < nJB) {
        // this CTA's last P1 product has released R1: the B panel of its first JB job goes out now; the job's h2 panel joins
        // the same mbarrier group after bar1.  W2t is written by the Adam phase and published by bar5; step 0 has no bar5
        // before it (the prologue's shadow writes are published by bar1), so step 0 issues the panel after bar1
        const int kt = cta % NTL;
        stage_block(st, R1, a.W2t + (size_t)kt * H * 32, H);
        w2t_pre = true;
      }
      float outv[4];
      tile_reduce<true, true>(acc, R0, outv);
      TR(4);
      {
        // 32 per-lane values (4 rows x MAXO products) -> lane l ends with the warp total of value l: a butterfly
        // that halves the value count at every step (31 shuffles, fixed order) instead of 5 shuffles per value
        float v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          v[r] = fmaxf(outv[r] + b2v, 0.f);
          a.h2[(size_t)(m0 + warp + 8 * r) * H + n0 + lane] = v[r];   // e = tid + r*256 -> (m = e >> 5, n = lane)
          a.h2t[((size_t)nt * B + m0 + warp + 8 * r) * 32 + lane] = v[r];   // and the tiled copy [H/32][B][32]
        }
        // value q = r * MAXO + o is v[r] * whr[o]; the first level pairs q with q + 16 as the products are formed, so
        // that only 16 values are ever live
        float hv_[16];
        const bool up16 = (lane & 16) != 0;
#pragma unroll
        for (int q = 0; q < 16; ++q) hv_[q] = butterfly_pair(v[q / MAXO] * whr[q % MAXO], v[q / MAXO + 2] * whr[q % MAXO], up16, 16);
        butterfly_level<8>(hv_, lane);
        butterfly_level<4>(hv_, lane);
        butterfly_level<2>(hv_, lane);
        butterfly_level<1>(hv_, lane);
        TR(35);
        const int r = lane >> 3, o = lane & 7;               // lane l holds value l = r * MAXO + o
        if (o < 4 * nq) a.headp[(((size_t)nt * 2 + (o >> 2)) * B + m0 + warp + 8 * r) * 4 + (o & 3)] = o < nout ? hv_[0] : 0.f;
      }
      row_ticket(mt, tid < 32, m0 + tid, tid);
    }
    xs_ready = false;
    TR(5);
    grid_bar(a.barrier, epoch, nctas);
    TR(6);

    // =========================== P3: critic means + backward jobs ======================================
    // the per-row table that the row tiles' last arrivers wrote before bar1: one bulk copy per CTA (d loss / d head outputs
    // into dsm, the second value-head candidate into dvs)
    stp.bytes = (unsigned)B * (MAXO + 1) * 4u;
    stp.commit();
    if (tid == 0) { stp.copy(dsm, a.dout, (unsigned)B * MAXO * 4u); stp.copy(dvs, a.dv2, (unsigned)B * 4u); }
    int pre_job = -1;                              // job whose first panels are already in flight
    if (cta < nJ3 && (cta < nJB || prefetchable(cta))) { issue_stage(cta, w2t_pre); pre_job = cta; }
    // tensor-core dh1 job: the first two W2^T chunks do not depend on the row maths, fetch them under the critic sums
    auto jb_issue_a = [&](int kt4, int nc, unsigned long long g) {
      const unsigned slot = (unsigned)(g % TC_NA);
      const unsigned bar = tc_bar + 8u * (TC_BAR_JB + slot), dst = tc_base + slot * TC_A_BYTES;
      mbar_expect_tx(bar, TC_A_BYTES);
      const float* src = a.W2Timg + ((size_t)kt4 * (H >> 5) + nc) * 4096;
      bulk_g2s(dst, src, 16384u, bar);
      bulk_g2s(dst + 16384u, src + (size_t)H * H, 16384u, bar);
    };
    if (TC && cta >= nJB && cta < nJB + nJA) {     // dW2 job: all minibatch rows' inputs, transposed [D][B]
      for (int e = tid; e < B * D; e += NT) { const int m = e / D, i = e - m * D; R2[i * B + m] = ldcg(a.xg + e); }
    }
    if (TC && cta < nJB && tid == 0) {
      jb_issue_a(cta / MT, 0, jb_g);
      if ((H >> 5) > 1) jb_issue_a(cta / MT, 1, jb_g + 1);
    }
    // row ids of the NEXT step's first P1 tile: the load is in flight during the whole phase
    const bool has_next = (s + 1 < a.n_steps) && cta < nJ1;
    int next_r = 0;
    if (TC) { if (has_next) next_r = a.perm[(cursor0 + s + 1) * (long long)B + (cta / NTL) * 128 + (tid & 127)]; }
    else if (has_next && tid < 32) next_r = a.perm[(cursor0 + s + 1) * (long long)B + (cta / NTL) * 32 + tid];

    float c1, c2;
    {
      // the per-row statistics, folded exactly as one thread per row (rows tid, tid + NT) and then the warps in order
      float p1 = 0.f, p2 = 0.f, ssum = 0.f, esum = 0.f, mr = -INFINITY, mp = INFINITY;
#pragma unroll 1
      for (int b = tid; b < B; b += NT) {
        const float d1 = ldcg(a.rowst + b), d2 = ldcg(a.rowst + B + b);
        p1 = fmaf(d1, d1, p1); p2 = fmaf(d2, d2, p2);   // one FMA per row: the rounding of the sums is fixed, not left to
                                                        // the compiler's mul/add contraction
        ssum += ldcg(a.rowst + 2 * B + b); esum += ldcg(a.rowst + 3 * B + b);
        mr = fmaxf(mr, ldcg(a.rowst + 4 * B + b)); mp = fminf(mp, ldcg(a.rowst + 5 * B + b));
      }
      p1 = jb_warp_sum(p1); p2 = jb_warp_sum(p2); ssum = jb_warp_sum(ssum); esum = jb_warp_sum(esum);
      mr = jb_warp_max(mr); mp = jb_warp_min(mp);
      if (lane == 0) { float* q = scr + warp * 8; q[0] = p1; q[1] = p2; q[2] = ssum; q[3] = esum; q[4] = mr; q[5] = mp; }
      __syncthreads();
      float t1 = 0.f, t2 = 0.f;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) { t1 += scr[w * 8]; t2 += scr[w * 8 + 1]; }
      float invBW = invB;
      if (a.world > 1) {
        // the two means of critic_loss = max(mean, mean) run over the GLOBAL minibatch (all ranks' rows): exchange the
        // row sums.  A peer's message for step s also says "I have finished step s-1", i.e. it no longer reads this
        // rank's gradient buffer, which the backward jobs below overwrite.
        const unsigned int target = a.xbase + (unsigned int)s + 1u;
        // message = two 8-byte words {row sum | tag}: an aligned 64-bit store is single-copy atomic, so payload and tag need
        // no fence between them (a release-signalled message cost microseconds per step); that the peer no longer READS this rank's
        // gradient follows from program order on the peer (its loads of step s-1 returned before it got here)
        unsigned long long m1 = 0ull, m2 = 0ull;
        if (tid < a.world && tid != a.rank) {
          if (cta == 0) {
            unsigned long long* dst = reinterpret_cast<unsigned long long*>(a.peer[tid] + a.xflag_off + JB_X_MSG + 4 * a.rank);
            const unsigned long long w1 = ((unsigned long long)target << 32) | (unsigned long long)__float_as_uint(t1);
            const unsigned long long w2 = ((unsigned long long)target << 32) | (unsigned long long)__float_as_uint(t2);
            asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(dst), "l"(w1) : "memory");
            asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(dst + 1), "l"(w2) : "memory");
          }
          const unsigned long long* src = reinterpret_cast<const unsigned long long*>(a.peer[a.rank] + a.xflag_off + JB_X_MSG + 4 * tid);
          const long long t0 = clock64();
          bool ok = false;
          while (!ok) {
            asm volatile("ld.relaxed.sys.global.u64 %0, [%1];\n" : "=l"(m1) : "l"(src) : "memory");
            asm volatile("ld.relaxed.sys.global.u64 %0, [%1];\n" : "=l"(m2) : "l"(src + 1) : "memory");
            ok = (int)((unsigned int)(m1 >> 32) - target) >= 0 && (int)((unsigned int)(m2 >> 32) - target) >= 0;
            if (!ok) {
              __nanosleep(50);
              unsigned int ab;
              asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(ab) : "l"(a.barrier + CTR_ABORT) : "memory");
              if (ab || clock64() - t0 > X_TIMEOUT_CYCLES) {
                asm volatile("st.relaxed.gpu.global.u32 [%0], %1;\n" ::"l"(a.barrier + CTR_ABORT), "r"(1u) : "memory");
                a.acc[7] = 1.f;
                if (cta == 0) { a.partials[200] = 3.f; a.partials[201] = (float)tid; a.partials[202] = (float)s; a.partials[203] = (float)(unsigned int)(m1 >> 32); a.partials[204] = (float)target; }
                break;
              }
            }
          }
          scr[96 + 2 * tid] = __uint_as_float((unsigned int)m1);      // peers' row sums, read by every thread below
          scr[96 + 2 * tid + 1] = __uint_as_float((unsigned int)m2);
        }
        __syncthreads();
        TR(40);
        float g1 = 0.f, g2 = 0.f;
        for (int r = 0; r < a.world; ++r) {                  // rank order: identical bits on every rank
          g1 += r == a.rank ? t1 : scr[96 + 2 * r];
          g2 += r == a.rank ? t2 : scr[96 + 2 * r + 1];
        }
        t1 = g1; t2 = g2;
        invBW = invB / (float)a.world;
      }
      c1 = t1 * invBW; c2 = t2 * invBW;
      float w1, w2;
      jbppo::critic_weights(c1, c2, w1, w2);
      stp.wait();
      TR(38);
      for (int b = tid; b < B; b += NT) dsm[b * MAXO + npol] = w1 * dsm[b * MAXO + npol] + w2 * dvs[b];
      if (cta == (int)nctas - 1 && tid == 0) {
        // learn()-level statistics of this minibatch (ppo.py:171-175), accumulated on the device
        float s3 = 0.f, s4 = 0.f, xr = -INFINITY, xp = INFINITY;
        for (int w = 0; w < NT / 32; ++w) { s3 += scr[w * 8 + 2]; s4 += scr[w * 8 + 3]; xr = fmaxf(xr, scr[w * 8 + 4]); xp = fminf(xp, scr[w * 8 + 5]); }
        a.acc[0] += -s3 * invB;
        a.acc[1] += fmaxf(c1, c2);
        a.acc[2] += -s4 * invB / (a.continuous ? (float)A : 1.f);
        a.acc[3] = fmaxf(a.acc[3], xr);
        a.acc[4] = fminf(a.acc[4], xp);
        a.acc[5] += 1.f;
      }
      __syncthreads();
    }
    TR(7);

    float sq = 0.f;                                // this thread's share of the step's squared gradient norm
    for (int job = cta; job < nJ3; job += (int)nctas) {
      __syncthreads();
      TR(8 + min(3, (job - cta) / (int)nctas));
      const int next = job + (int)nctas;
      if (TC && job < nJB) {
        // ---- tensor-core dh1 job: D[128 hidden units k][32 rows m] = sum_n W2[n][k] dh2[m][n]  (dh1 transposed) ---------
        // A chunk = hi | lo image of W2^T [128 k][32 n] (two 16 KB bulk copies, two chunks ahead); B chunk = dh2^T
        // [32 m][32 n] = ((dout Wh) * relu'(h2)) generated by the threads, ONE float4 each; 4 x 3 wgmma per chunk and warpgroup.
        // Epilogue: mask by relu'(h1) (h1 recomputed from x: D FMAs), partial dW1 / db1 of this 32-row tile.
        const int kt4 = job / MT, mt = job - kt4 * MT, m0 = mt * 32, kin0 = kt4 * 128, NKC = H >> 5;
        if (job != cta && tid == 0) {
          jb_issue_a(kt4, 0, jb_g);
          if (NKC > 1) jb_issue_a(kt4, 1, jb_g + 1);
        }
        for (int e = tid; e < 32 * MAXD; e += NT) { const int r = e >> 4, i = e & 15; xs[i * 32 + r] = i < D ? ldcg(a.xg + (size_t)(m0 + r) * D + i) : 0.f; }
        const int ml = tid >> 3, c8 = tid & 7;                      // this thread's element group: row m0 + ml, columns 4 c8 .. + 3 of a chunk
        const float* drow = &dsm[(m0 + ml) * MAXO];
        float4 hq = ldcg4(a.h2 + (size_t)(m0 + ml) * H + 4 * c8);     // h2 of chunk 0 (prefetched one chunk ahead below)
        float acc[16];
        for (int nc = 0; nc < NKC; ++nc) {
          const unsigned long long g = jb_g + nc;
          const unsigned slot = (unsigned)(g % TC_NA);                 // B slot of chunk g - 3: retired (wait below)
          float4 wr[MAXO];
#pragma unroll
          for (int o = 0; o < MAXO; ++o) wr[o] = o < nout ? *reinterpret_cast<const float4*>(&PS[o * PK + nc * 32 + 4 * c8]) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 hcur = hq;
          if (nc + 1 < NKC) hq = ldcg4(a.h2 + (size_t)(m0 + ml) * H + (nc + 1) * 32 + 4 * c8);
          const float4 dv = dh2_quad<NO>(drow, wr, hcur);
          const float4 lo = make_float4(tf32_lo(dv.x), tf32_lo(dv.y), tf32_lo(dv.z), tf32_lo(dv.w));
          const unsigned bbuf = tc_base + TC_NA * TC_A_BYTES + slot * TC_B_BYTES, off = tile_off(ml, c8);
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(bbuf + off), "f"(dv.x), "f"(dv.y), "f"(dv.z), "f"(dv.w) : "memory");
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(bbuf + 4096u + off), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
          jbwg::wait<0>();                                              // chunk g - 1's products of this warpgroup retired
          jbwg::fence_acc(acc);
          asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
          __syncthreads();                                              // ... and those of the other warpgroup
          if (tid == 0 && nc + 2 < NKC) jb_issue_a(kt4, nc + 2, g + 2);  // A ring: chunk nc + 2 goes where chunk nc - 1 lived
          mbar_wait(tc_bar + 8u * (TC_BAR_JB + slot), (unsigned)((g / TC_NA) & 1));   // W2^T chunk landed
          const unsigned aw = tc_base + slot * TC_A_BYTES + (unsigned)wg * 8192u;
          jbwg::fence();
          jbwg::mma3_n32(acc, aw, aw + 16384u, bbuf, bbuf + 4096u, nc == 0);
          jbwg::commit();
        }
        jbwg::wait<0>();
        jbwg::fence_acc(acc);
        __syncthreads();                                          // both warpgroups' products retired: tcs overlays A slot 1
        jbwg::store_acc_n32(acc, tcs, TC_LD);
        __syncthreads();
        if (prefetchable(next)) { issue_stage(next, false); pre_job = next; }   // every MMA that read the rings has retired
        {
          const int q = warp & 3, cb = (warp >> 2) * 16, kin = kin0 + q * 32 + lane;
          float rr[16];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 t = *reinterpret_cast<const float4*>(&tcs[(q * 32 + lane) * TC_LD + cb + 4 * c]);
            rr[4 * c] = t.x; rr[4 * c + 1] = t.y; rr[4 * c + 2] = t.z; rr[4 * c + 3] = t.w;
          }
          // h1[m][kin] > 0 ?  (same arithmetic as the forward phase: fma chain over the inputs, then + b1)
          float w1r[ND];
#pragma unroll
          for (int i = 0; i < ND; ++i) w1r[i] = i < D ? ldcg(a.W1 + (size_t)kin * D + i) : 0.f;
          const float b1v = PS[(MAXO + 1) * PK + kin];
          float wacc[ND + 1];
#pragma unroll
          for (int i = 0; i <= ND; ++i) wacc[i] = 0.f;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int ml2 = cb + j;
            float h = 0.f;
#pragma unroll
            for (int i = 0; i < ND; ++i) if (i < D) h = fmaf(xs[i * 32 + ml2], w1r[i], h);
            const float dvv = (h + b1v > 0.f) ? rr[j] : 0.f;
#pragma unroll
            for (int i = 0; i < ND; ++i) if (i < D) wacc[i] = fmaf(dvv, xs[i * 32 + ml2], wacc[i]);
            wacc[ND] += dvv;
          }
          float* sc = tcp + (size_t)(q * 32 + lane) * (MAXD + 1);       // [128 k][MAXD + 1] scratch in ring slot 0
          if (warp >= 4) {
#pragma unroll
            for (int i = 0; i <= ND; ++i) if (i < D || i == ND) sc[i < D ? i : MAXD] = wacc[i];
          }
          __syncthreads();
          if (warp < 4) {
            float* dstw = a.w1p + ((size_t)mt * H + kin) * (D + 1);
#pragma unroll
            for (int i = 0; i < ND; ++i) if (i < D) dstw[i] = wacc[i] + sc[i];
            dstw[D] = wacc[ND] + sc[MAXD];
          }
          __syncthreads();
        }
        if (tid < 4) asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(a.barrier + CTR_JB + kt4 * 4 + tid) : "memory");
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // scratch reads above before later bulk copies / wgmma
        jb_g += (unsigned long long)NKC;
        TR(16);
      } else if (!TC && job < nJB) {
        // ---- dh1 tile = ((dout Wh) * relu'(h2)) W2, masked by relu'(h1); partial dW1 / db1 ---------------
        const int mt = job / NTL, kt = job - mt * NTL;
        const int m0 = mt * 32, k0 = kt * 32;
        if (pre_job != job) issue_stage(job, false);
        const int c4 = (tid & 127) * 4, rh = tid >> 7;
        float4 wr[MAXO];
#pragma unroll
        for (int o = 0; o < MAXO; ++o)
          wr[o] = (o < nout && c4 < H) ? *reinterpret_cast<const float4*>(&PS[o * PK + c4]) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (TC || !(job == cta && nJ1 <= (int)nctas))    // else xs still holds these rows from this CTA's P1 tile
          for (int e = tid; e < 32 * MAXD; e += NT) { const int r = e >> 4, i = e & 15; xs[i * 32 + r] = i < D ? ldcg(a.xg + (size_t)(m0 + r) * D + i) : 0.f; }
        float h1m[4];                              // relu mask of the output tile: asm volatile keeps the loads HERE
#pragma unroll
        for (int r = 0; r < 4; ++r)
          asm volatile("ld.global.cg.f32 %0, [%1];\n" : "=f"(h1m[r]) : "l"(a.h1 + ((size_t)kt * B + m0 + warp + 8 * r) * 32 + lane));
        st.wait();
        TR(12);
        if (c4 < H) {
#pragma unroll 4
          for (int r = 0; r < 16; ++r) {
            const int row = rh * 16 + r;
            float4* pa = reinterpret_cast<float4*>(&R0[row * (H + 4) + c4]);
            *pa = dh2_quad<NO>(&dsm[(m0 + row) * MAXO], wr, *pa);
          }
        }
        __syncthreads();
        TR(13);
        float acc[8][8] = {};
        tile_mma<true, false>(R0, R1, H, acc, nullptr);
        __syncthreads();
        TR(14);
        if (prefetchable(next)) { issue_stage(next, false); pre_job = next; }
        float outv[4];
        tile_reduce<true, false>(acc, R0, outv);
        TR(15);
        // partial dW1[k0+n][i] = sum_{m in tile} dh1[m, n] x[m, i], db1 likewise: 4 rows per thread, then 8 warps
        float wacc[MAXD + 1];
#pragma unroll
        for (int i = 0; i <= MAXD; ++i) wacc[i] = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float dv = h1m[r] > 0.f ? outv[r] : 0.f;
          const float* xrow = &xs[warp + 8 * r];
#pragma unroll
          for (int i = 0; i < MAXD; ++i) if (i < D) wacc[i] = fmaf(dv, xrow[i * 32], wacc[i]);
          wacc[MAXD] += dv;
        }
        __syncthreads();                           // the fold's reads of R0 are done
#pragma unroll
        for (int i = 0; i <= MAXD; ++i) if (i < D || i == MAXD) R0[(warp * (MAXD + 1) + i) * 32 + lane] = wacc[i];
        __syncthreads();
        TR(33);
        for (int e = tid; e < 32 * (D + 1); e += NT) {
          const int n = e / (D + 1), i = e - n * (D + 1);
          const int slot = i < D ? i : MAXD;
          float t = R0[(0 * (MAXD + 1) + slot) * 32 + n];
#pragma unroll
          for (int w = 1; w < NT / 32; ++w) t += R0[(w * (MAXD + 1) + slot) * 32 + n];
          a.w1p[((size_t)mt * H + k0) * (D + 1) + e] = t;
        }
        __syncthreads();
        TR(34);
        if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(a.barrier + CTR_JB + kt) : "memory");
        TR(16);
      } else if (TC && job < nJB + nJA) {
        // ---- tensor-core dW2 job: D[128 k][32 n] = sum_m h1[m][k] dh2[m][n]  (a tile of dW2^T), K = minibatch rows in chunks of 32.
        // Both operands are GENERATED: A chunk = h1^T [128 k][32 m] = relu(x W1^T + b1) (thread = one k, 16 rows),
        // B chunk = dh2^T [32 n][32 m] (thread = one n, 4 rows); db2 = row sums of the B operand (jobs of k-tile 0).
        const int j = job - nJB, kt4 = j / NTL, nt = j - kt4 * NTL, k0 = kt4 * 128, n0 = nt * 32, NMC = B >> 5;
        float* xall = R2;                                          // [D][B]
        if (job != cta) {
          __syncthreads();
          for (int e = tid; e < B * D; e += NT) { const int m = e / D, i = e - m * D; xall[i * B + m] = ldcg(a.xg + e); }
        }
        const int r = tid & 127, half = tid >> 7;                  // A: hidden unit k0 + r, rows 16 half .. + 15 of a chunk
        float w1r[ND];
#pragma unroll
        for (int i = 0; i < ND; ++i) w1r[i] = i < D ? ldcg(a.W1 + (size_t)(k0 + r) * D + i) : 0.f;
        const float b1v = PS[(MAXO + 1) * PK + k0 + r];
        const int nl = tid >> 3, c8 = tid & 7;                     // B: hidden unit n0 + nl, rows 4 c8 .. + 3 of a chunk
        float whn[MAXO];
#pragma unroll
        for (int o = 0; o < MAXO; ++o) whn[o] = o < nout ? PS[o * PK + n0 + nl] : 0.f;
        const float* h2col = a.h2t + (size_t)nt * B * 32 + nl;      // h2[m][n0 + nl] = h2col[m * 32]
        float hq[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) hq[q] = ldcg(h2col + (size_t)(4 * c8 + q) * 32);
        float b2acc = 0.f;
        float acc[16];
        __syncthreads();                                            // xall complete
        for (int mc = 0; mc < NMC; ++mc) {
          const unsigned long long g = ja_g + mc;
          const unsigned slot = (unsigned)(g % TC_NA);              // slots of chunk g - 3: retired (wait below)
          const unsigned abuf = tc_base + slot * TC_A_BYTES, bbuf = tc_base + TC_NA * TC_A_BYTES + slot * TC_B_BYTES;
          // A chunk
          float hv[16];
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) hv[jj] = 0.f;
#pragma unroll
          for (int i = 0; i < ND; ++i) {
            if (i < D) {
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const float4 x4 = *reinterpret_cast<const float4*>(&xall[i * B + mc * 32 + half * 16 + 4 * c]);
                hv[4 * c] = fmaf(x4.x, w1r[i], hv[4 * c]); hv[4 * c + 1] = fmaf(x4.y, w1r[i], hv[4 * c + 1]);
                hv[4 * c + 2] = fmaf(x4.z, w1r[i], hv[4 * c + 2]); hv[4 * c + 3] = fmaf(x4.w, w1r[i], hv[4 * c + 3]);
              }
            }
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const unsigned off = tile_off(r, half * 4 + c);
            const float4 hi = make_float4(fmaxf(hv[4 * c] + b1v, 0.f), fmaxf(hv[4 * c + 1] + b1v, 0.f), fmaxf(hv[4 * c + 2] + b1v, 0.f), fmaxf(hv[4 * c + 3] + b1v, 0.f));
            const float4 lo = make_float4(tf32_lo(hi.x), tf32_lo(hi.y), tf32_lo(hi.z), tf32_lo(hi.w));
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(abuf + off), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(abuf + 16384u + off), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
          }
          // B chunk
          {
            float hc[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) hc[q] = hq[q];
            if (mc + 1 < NMC) {
#pragma unroll
              for (int q = 0; q < 4; ++q) hq[q] = ldcg(h2col + (size_t)((mc + 1) * 32 + 4 * c8 + q) * 32);
            }
            float dv[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float* d = &dsm[(mc * 32 + 4 * c8 + q) * MAXO];
              const float4 d0 = *reinterpret_cast<const float4*>(d), d1 = *reinterpret_cast<const float4*>(d + 4);
              float t = d0.x * whn[0];
              t = fmaf(d0.y, whn[1], t); t = fmaf(d0.z, whn[2], t); t = fmaf(d0.w, whn[3], t);
              t = fmaf(d1.x, whn[4], t); t = fmaf(d1.y, whn[5], t); t = fmaf(d1.z, whn[6], t); t = fmaf(d1.w, whn[7], t);
              dv[q] = hc[q] > 0.f ? t : 0.f;                        // same arithmetic as dh2_quad
            }
            b2acc += (dv[0] + dv[1]) + (dv[2] + dv[3]);
            const unsigned off = tile_off(nl, c8);
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(bbuf + off), "f"(dv[0]), "f"(dv[1]), "f"(dv[2]), "f"(dv[3]) : "memory");
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(bbuf + 4096u + off), "f"(tf32_lo(dv[0])), "f"(tf32_lo(dv[1])), "f"(tf32_lo(dv[2])), "f"(tf32_lo(dv[3])) : "memory");
          }
          jbwg::wait<0>();                                          // chunk g - 1's products of this warpgroup retired
          jbwg::fence_acc(acc);
          asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
          __syncthreads();                                          // ... and those of the other warpgroup
          const unsigned aw = abuf + (unsigned)wg * 8192u;
          jbwg::fence();
          jbwg::mma3_n32(acc, aw, aw + 16384u, bbuf, bbuf + 4096u, mc == 0);
          jbwg::commit();
        }
        jbwg::wait<0>();
        jbwg::fence_acc(acc);
        __syncthreads();                                          // both warpgroups' products retired: tcs overlays A slot 1
        jbwg::store_acc_n32(acc, tcs, TC_LD);
        __syncthreads();
        {
          const int q = warp & 3, cb = (warp >> 2) * 16, kk = k0 + q * 32 + lane;
          float rr[16];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 t = *reinterpret_cast<const float4*>(&tcs[(q * 32 + lane) * TC_LD + cb + 4 * c]);
            rr[4 * c] = t.x; rr[4 * c + 1] = t.y; rr[4 * c + 2] = t.z; rr[4 * c + 3] = t.w;
          }
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float v = rr[i];
            a.gW2[(size_t)(n0 + cb + i) * H + kk] = v;              // lanes = consecutive k: 128-byte rows
            sq = fmaf(v, v, sq);
          }
          if (kt4 == 0) {                                          // db2[n] = sum over all rows: fold the 8 row groups of hidden unit nl
            float t = b2acc;
            t += __shfl_xor_sync(0xffffffffu, t, 1); t += __shfl_xor_sync(0xffffffffu, t, 2); t += __shfl_xor_sync(0xffffffffu, t, 4);
            if (c8 == 0) { a.gb2[n0 + nl] = t; sq = fmaf(t, t, sq); }
          }
          asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
          __syncthreads();
        }
        ja_g += (unsigned long long)NMC;
        TR(21);
      } else if (!TC && job < nJB + nJA) {
        // ---- a pair of dW2 tiles [n0.., k0..] = sum_m dh2[m, n] h1[m, k] sharing the dh2 panel; db2 = its row sums
        const int j = job - nJB;
        const int nt = j / NP, kt0 = 2 * (j - nt * NP);
        const int n0 = nt * 32;
        const int cg = tid & 7, rl = tid >> 3;
        float4 wr[MAXO];
#pragma unroll
        for (int o = 0; o < MAXO; ++o) wr[o] = o < nout ? *reinterpret_cast<const float4*>(&PS[o * PK + n0 + 4 * cg]) : make_float4(0.f, 0.f, 0.f, 0.f);
        const int nhalf = (kt0 + 1 < NTL) ? 2 : 1;
        for (int half = 0; half < nhalf; ++half) {
          const int kt = kt0 + half, k0 = kt * 32;
          const float* Bp = R1 + ((single && half == 1) ? R2_FLOATS : 0);
          float acc[8][8] = {};
          float rs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          for (int mp = 0; mp < B; mp += JA_ROWS) {
            const int kp = min(JA_ROWS, B - mp);
            if (!single || half == 0) {
              if (single) {
                if (pre_job != job) issue_stage(job, false);
              } else {
                __syncthreads();
                stage_block(st, R2, a.h2t + ((size_t)nt * B + mp) * 32, kp);
                stage_block(st, R1, a.h1 + ((size_t)kt * B + mp) * 32, kp);
                st.commit();
              }
              st.wait();
              TR(17);
              for (int m = rl; m < kp; m += 32) {
                float4* pa = reinterpret_cast<float4*>(&R2[m * 32 + 4 * cg]);
                *pa = dh2_quad<NO>(&dsm[(mp + m) * MAXO], wr, *pa);
              }
              __syncthreads();
              TR(18);
            }
            tile_mma<false, false>(R2, Bp, kp, acc, kt == 0 ? rs : nullptr);
          }
          __syncthreads();
          TR(19);
          if (half == nhalf - 1 && prefetchable(next)) { issue_stage(next, false); pre_job = next; }
          float outv[4];
          tile_reduce<false, false>(acc, R0, outv);
          TR(20);
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            a.gW2[(size_t)(n0 + warp + 8 * r) * H + k0 + lane] = outv[r];
            sq = fmaf(outv[r], outv[r], sq);
          }
          if (kt == 0) {
            const int grp = tid >> 4, t = tid & 15, tx = t & 3, ty = t >> 2;
            __syncthreads();                       // the fold's reads of R0 are done
            if (tx == 0) {
#pragma unroll
              for (int i = 0; i < 8; ++i) R0[grp * 32 + ty * 8 + i] = rs[i];
            }
            __syncthreads();
            if (tid < 32) {
              float v = 0.f;
#pragma unroll
              for (int g = 0; g < KG; ++g) v += R0[g * 32 + tid];
              a.gb2[n0 + tid] = v;
              sq = fmaf(v, v, sq);
            }
            __syncthreads();
          }
        }
        TR(21);
      } else if (job < nJB + nJA + nJC) {
        // ---- head weight gradients, 32 columns per job; job 0 also the head bias gradients -------------
        const int jt = job - nJB - nJA;
        const int j0 = jt * 32;   // first column of the tile
        float hacc[MAXO];
#pragma unroll
        for (int o = 0; o < MAXO; ++o) hacc[o] = 0.f;
        for (int mp = 0; mp < B; mp += JA_ROWS) {
          const int kp = min(JA_ROWS, B - mp);
          if (!(mp == 0 && pre_job == job)) { __syncthreads(); stage_block(st, R2, a.h2t + ((size_t)jt * B + mp) * 32, kp); st.commit(); }
          st.wait();
          if (!TC) TR(39);                 // (JC / JD stamps: FFMA engine only, they cost the tensor-core instantiations spills)
#pragma unroll 4
          for (int m = warp; m < kp; m += NT / 32) {
            const float hvv = R2[m * 32 + lane];
            const float4 d0 = *reinterpret_cast<const float4*>(&dsm[(mp + m) * MAXO]);
            const float4 d1 = *reinterpret_cast<const float4*>(&dsm[(mp + m) * MAXO + 4]);
            hacc[0] = fmaf(d0.x, hvv, hacc[0]); hacc[1] = fmaf(d0.y, hvv, hacc[1]); hacc[2] = fmaf(d0.z, hvv, hacc[2]);
            hacc[3] = fmaf(d0.w, hvv, hacc[3]); hacc[4] = fmaf(d1.x, hvv, hacc[4]); hacc[5] = fmaf(d1.y, hvv, hacc[5]);
            hacc[6] = fmaf(d1.z, hvv, hacc[6]); hacc[7] = fmaf(d1.w, hvv, hacc[7]);
          }
        }
        __syncthreads();
        if (prefetchable(next)) { issue_stage(next, false); pre_job = next; }
        float* red = R0;               // [8][MAXO][32]
#pragma unroll
        for (int o = 0; o < MAXO; ++o) red[(warp * MAXO + o) * 32 + lane] = hacc[o];
        __syncthreads();
        if (warp == 0) {
#pragma unroll
          for (int o = 0; o < MAXO; ++o) {
            if (o < nout) {
              float t = red[(0 * MAXO + o) * 32 + lane];
              for (int r = 1; r < NT / 32; ++r) t += red[(r * MAXO + o) * 32 + lane];
              ht.gw[o][j0 + lane] = t;
              sq = fmaf(t, t, sq);
            }
          }
        }
        if (jt == 0) {
          // bias gradients db[o] = sum_m dout[m][o]: 32 partial sums per output, folded in a fixed order
          __syncthreads();
          const int o = tid & 7, part = tid >> 3;
          float t = 0.f;
          for (int m = part; m < B; m += NT / 8) t += dsm[m * MAXO + o];
          red[part * MAXO + o] = t;
          __syncthreads();
          if (tid < MAXO) {
            float tt = 0.f;
            for (int q = 0; q < NT / 8; ++q) tt += red[q * MAXO + tid];
            if (tid < nout) { *ht.gb[tid] = tt; sq = fmaf(tt, tt, sq); }
          }
        }
        if (!TC) TR(30);
      } else {
        // ---- dW1 / db1 of 32 hidden units: fixed-order fold of the MT tile partials ----------------------
        const int kt = job - nJB - nJA - nJC, k0 = kt * 32;
        if (tid == 0) {
          const unsigned int target = (unsigned int)MT * (unsigned int)(s + 1);
          unsigned int v;
          do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(a.barrier + CTR_JB + kt) : "memory");
          } while (v < target);
          asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
        }
        __syncthreads();
        if (!TC) TR(31);
        for (int e = tid; e < 32 * (D + 1); e += NT) {
          const int n = e / (D + 1), i = e - n * (D + 1);
          float t = ldcg(a.w1p + (size_t)k0 * (D + 1) + e);
          for (int mt = 1; mt < MT; ++mt) t += ldcg(a.w1p + ((size_t)mt * H + k0) * (D + 1) + e);
          if (i < D) a.gW1[(size_t)(k0 + n) * D + i] = t; else a.gb1[k0 + n] = t;
          sq = fmaf(t, t, sq);
        }
        if (!TC) TR(32);
      }
    }
    TR(22);
    if (a.world == 1) {                            // (multi-GPU: the norm is taken of the AVERAGED gradient, below)
      const float tot = block_sum(sq, scr + 64);
      if (tid == 0) a.partials[cta] = tot;
    }
    if (!TC && has_next && tid < 32) sidx[tid] = next_r;
    // Adam operands that do not depend on this step's gradient: in registers across the barrier
    float4 pp[ADAM_IT], mm[ADAM_IT], vv[ADAM_IT];
#pragma unroll
    for (int it = 0; it < ADAM_IT; ++it) {
      const long long i = lo + tid + it * NT;
      if (i < hi) { pp[it] = __ldcg(p4 + i); mm[it] = __ldcg(m4 + i); vv[it] = __ldcg(v4 + i); }
    }
    TR(23);
    grid_bar(a.barrier, epoch, nctas);
    TR(24);

    // =========================== P5: clip + Adam on this CTA's slice ===================================
    {
      float4 gg[ADAM_IT];
      if (a.world == 1) {
#pragma unroll
        for (int it = 0; it < ADAM_IT; ++it) {
          const long long i = lo + tid + it * NT;
          if (i < hi) gg[it] = __ldcg(g4 + i);
        }
      } else {
        // ---- gradient average over peer memory (NVLink): reduce-scatter to the slice owners + all-gather, both as LL words
        const unsigned int target = a.xbase + (unsigned int)s + 1u;
        unsigned int* abortf = a.barrier + CTR_ABORT;
        const long long q4 = (a.P4 + a.world - 1) / a.world, c4 = (q4 + nctas - 1) / nctas;
        bool ok = true;
        // (1) push: this CTA's chunk of every OTHER owner's slice of the local gradient -> that owner's inbox [src = me]
        for (int q = 0; q < a.world; ++q) {
          if (q == a.rank) continue;
          const long long sl_lo = (long long)q * q4, sl_hi = min(a.P4, sl_lo + q4);
          const long long ch_lo = sl_lo + (long long)cta * c4, ch_hi = min(sl_hi, ch_lo + c4);
          unsigned long long* inbox = reinterpret_cast<unsigned long long*>(a.peer[q] + a.xllin_off) + ((size_t)a.rank * q4) * 4;
          for (long long i = ch_lo + tid; i < ch_hi; i += NT) ll_store4(inbox + (i - sl_lo) * 4, __ldcg(g4 + i), target);
        }
        TR(41);
        {
          // (2) this CTA owns chunk `cta` of slice `rank`: sum the ranks' copies in rank order (the same bits whoever owns the
          // chunk), scale, and send the averaged chunk to every rank's copy of the averaged gradient
          const long long sl_lo = (long long)a.rank * q4, sl_hi = min(a.P4, sl_lo + q4);
          const long long ch_lo = sl_lo + (long long)cta * c4, ch_hi = min(sl_hi, ch_lo + c4);
          const unsigned long long* inbox = reinterpret_cast<const unsigned long long*>(a.peer[a.rank] + a.xllin_off);
          const float inv_world = 1.f / (float)a.world;
          float sqa = 0.f;
          for (long long i = ch_lo + tid; i < ch_hi; i += NT) {
            float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < a.world; ++r) {
              float4 t;
              if (r == a.rank) t = __ldcg(g4 + i);
              else ok = ll_load4(inbox + ((size_t)r * q4 + (i - sl_lo)) * 4, target, t, abortf) && ok;
              sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
            }
            sum.x *= inv_world; sum.y *= inv_world; sum.z *= inv_world; sum.w *= inv_world;
            sqa = fmaf(sum.x, sum.x, sqa); sqa = fmaf(sum.y, sum.y, sqa); sqa = fmaf(sum.z, sum.z, sqa); sqa = fmaf(sum.w, sum.w, sqa);
            for (int r = 0; r < a.world; ++r)
              ll_store4(reinterpret_cast<unsigned long long*>(a.peer[r] + a.xgred_off) + (size_t)i * 4, sum, target);
          }
          const float tot = block_sum(sqa, scr + 64);
          TR(42);
          if (tid < a.world) {                                        // the chunk's squared norm, one LL word per destination rank
            unsigned long long* pt = reinterpret_cast<unsigned long long*>(a.peer[tid] + a.xflag_off + JB_X_PTAB) + (a.rank * JB_X_MAX_CTAS + cta);
            asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(pt), "l"(ll_pack(tot, target)) : "memory");
          }
        }
        TR(43);
        // (3) this CTA's Adam slice of the averaged gradient (words arrive from all owners), and all chunk norms
        const unsigned long long* avg = reinterpret_cast<const unsigned long long*>(a.peer[a.rank] + a.xgred_off);
#pragma unroll
        for (int it = 0; it < ADAM_IT; ++it) {
          const long long i = lo + tid + it * NT;
          if (i < hi) ok = ll_load4(avg + (size_t)i * 4, target, gg[it], abortf) && ok;
        }
        if (tid < (int)nctas) {
          const unsigned long long* pt = reinterpret_cast<const unsigned long long*>(a.peer[a.rank] + a.xflag_off + JB_X_PTAB);
          float t = 0.f;
          for (int r = 0; r < a.world; ++r) {                         // owner-rank order
            float v;
            ok = ll_load1(pt + (r * JB_X_MAX_CTAS + tid), target, v, abortf) && ok;
            t += v;
          }
          dvs[tid] = t;
        }
        if (!ok) {
          a.acc[7] = 1.f;
          if (cta == 0) { a.partials[200] = 1.f; a.partials[201] = (float)tid; a.partials[202] = (float)s; a.partials[204] = (float)target; }
        }
        TR(44);
      }
      // next step's state rows (sidx was published before the barrier)
      float xv[2] = {0.f, 0.f};
      if (TC) {
        if (has_next) {
          xpre_idx = next_r;
#pragma unroll
          for (int i = 0; i < ND; ++i) if (i < D) xpre[i] = a.state[(size_t)next_r * D + i];
        }
      } else if (has_next) {
#pragma unroll
        for (int q = 0; q < 2; ++q) { const int e = tid + q * NT, r = e >> 4, i = e & 15; if (i < D) xv[q] = a.state[(size_t)sidx[r] * D + i]; }
      }
      // ||g||: one coalesced read of the partials per CTA, then every warp folds them in the same fixed order
      if (a.world == 1 && tid < (int)nctas) dvs[tid] = ldcg(a.partials + tid);     // (multi-GPU: filled by the exchange above)
      __syncthreads();
      float pv[NT / 32];
#pragma unroll
      for (int q = 0; q < NT / 32; ++q) pv[q] = lane + 32 * q < (int)nctas ? dvs[lane + 32 * q] : 0.f;
      double t = 0.0;
#pragma unroll
      for (int q = 0; q < NT / 32; ++q) t += (double)pv[q];
      t = jb_warp_sum_d(t);
      const float total_norm = (float)sqrt(t);
      float coef = 1.f;
      if (a.max_norm > 0.f) { coef = a.max_norm / (total_norm + 1e-6f); coef = coef < 1.f ? coef : 1.f; }
      const float step_size = (float)((double)lr / (1.0 - pw1));
      const float bc2_sqrt = (float)sqrt(1.0 - pw2);
      pw1 *= (double)a.beta1; pw2 *= (double)a.beta2;
      TR(25);
      // sqrt / reciprocal by the MUFU approximations (<= 2 ulp): the quotient only scales a term that is
      // ~lr times smaller than the parameter it is added to, so the rounding of p is unchanged to ~1e-11
      const float inv_bc2 = 1.f / bc2_sqrt;
      auto upd = [&](float& p_, float g_, float& m_, float& v_) {
        g_ *= coef;
        m_ = fmaf(g_ - m_, one_m_b1, m_);
        v_ = fmaf(one_m_b2 * g_, g_, a.beta2 * v_);
        float sq_, rc_;
        asm("sqrt.approx.f32 %0, %1;" : "=f"(sq_) : "f"(v_));
        const float denom = fmaf(sq_, inv_bc2, a.adam_eps);
        asm("rcp.approx.f32 %0, %1;" : "=f"(rc_) : "f"(denom));
        p_ = fmaf(-step_size, m_ * rc_, p_);
      };
#pragma unroll
      for (int it = 0; it < ADAM_IT; ++it) {
        const long long i = lo + tid + it * NT;
        if (i < hi) {
          upd(pp[it].x, gg[it].x, mm[it].x, vv[it].x); upd(pp[it].y, gg[it].y, mm[it].y, vv[it].y);
          upd(pp[it].z, gg[it].z, mm[it].z, vv[it].z); upd(pp[it].w, gg[it].w, mm[it].w, vv[it].w);
          p4[i] = pp[it]; m4[i] = mm[it]; v4[i] = vv[it];
          shadow(i, pp[it]);
        }
      }
      for (long long i = lo + tid + (long long)ADAM_IT * NT; i < hi; i += NT) {   // slices beyond 4 K floats per CTA
        float4 p_ = __ldcg(p4 + i), m_ = __ldcg(m4 + i), v_ = __ldcg(v4 + i);
        float4 g_;
        if (a.world > 1) {
          if (!ll_load4(reinterpret_cast<const unsigned long long*>(a.peer[a.rank] + a.xgred_off) + (size_t)i * 4, a.xbase + (unsigned int)s + 1u, g_, a.barrier + CTR_ABORT)) a.acc[7] = 1.f;
        } else g_ = __ldcg(g4 + i);
        upd(p_.x, g_.x, m_.x, v_.x); upd(p_.y, g_.y, m_.y, v_.y); upd(p_.z, g_.z, m_.z, v_.z); upd(p_.w, g_.w, m_.w, v_.w);
        p4[i] = p_; m4[i] = m_; v4[i] = v_;
        shadow(i, p_);
      }
      if (has_next) {
        if (!TC) {
#pragma unroll
          for (int q = 0; q < 2; ++q) { const int e = tid + q * NT; xs[(e & 15) * 32 + (e >> 4)] = xv[q]; }
        }
        xs_ready = true;
      }
    }
    TR(26);
    grid_bar(a.barrier, epoch, nctas);
    TR(27);
  }
  if (cta == 0 && tid == 0) { *a.step = step0 + a.n_steps; *a.cursor = cursor0 + a.n_steps; }
}

static int dsm_floats_for(int B) { return B * MAXO; }
static size_t fused_smem(int B) { return sizeof(float) * (size_t)(SMALL_FLOATS + dsm_floats_for(B) + 2 * RED_FLOATS + R2_FLOATS + PS_FLOATS); }

// Largest grid the cooperative launch can keep co-resident (one CTA per SM) for minibatch size B.
static const void* fused_fn(bool tc, int A, int D) {
  const int na = A <= 2 ? 0 : (A <= 4 ? 1 : 2), nd = D <= 4 ? 0 : 1;
  static const void* const tab[4][3] = {
      {(const void*)ppo_epoch_kernel<false, 2, 4>, (const void*)ppo_epoch_kernel<false, 4, 4>, (const void*)ppo_epoch_kernel<false, 8, 4>},
      {(const void*)ppo_epoch_kernel<false, 2, 16>, (const void*)ppo_epoch_kernel<false, 4, 16>, (const void*)ppo_epoch_kernel<false, 8, 16>},
      {(const void*)ppo_epoch_kernel<true, 2, 4>, (const void*)ppo_epoch_kernel<true, 4, 4>, (const void*)ppo_epoch_kernel<true, 8, 4>},
      {(const void*)ppo_epoch_kernel<true, 2, 16>, (const void*)ppo_epoch_kernel<true, 4, 16>, (const void*)ppo_epoch_kernel<true, 8, 16>}};
  return tab[(tc ? 2 : 0) + nd][na];
}

static int fused_max_ctas(int B, bool tc = false, int A = 8, int D = 16) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t smem = fused_smem(B);
  if (smem > 227 * 1024) return 0;
  const void* fn = fused_fn(tc, A, D);
  cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, NT, smem);
  return sms * (per_sm > 0 ? 1 : 0);
}

}  // namespace

JB_API int jb_ppo_fused_args_size(void) { return (int)sizeof(jb_ppo_fused_args); }

JB_API int jb_ppo_fused_max_ctas(void) { return fused_max_ctas(256); }

// Debug: copy the clock64 trace of the last step (JB_FUSED_SKIP=256) to host memory: [256 CTAs][48 slots].
JB_API int jb_ppo_fused_trace(long long* host_out) {
  return cudaMemcpyFromSymbol(host_out, g_trace, sizeof(long long) * 256 * 48) == cudaSuccess ? JB_OK : JB_ERR_CUDA;
}

// Runs args->n_steps minibatch steps starting at the device-side cursor.  `args` is a HOST pointer to
// a jb_ppo_fused_args (include/jorldy_b200_fused.h); it is copied at launch.
JB_API int jb_ppo_fused_run(const void* host_args, void* stream) {
  if (!host_args) return JB_ERR_INVALID;
  Args a = *reinterpret_cast<const Args*>(host_args);
  if (a.B <= 0 || a.B % 32 || a.B > MAX_B || a.H <= 0 || a.H % 32 || a.H > PK || a.D <= 0 || a.D > MAXD || a.nout <= 0 ||
      a.nout > MAXO || a.A <= 0 || a.A > jbppo::MAX_A || a.n_steps <= 0 || a.P4 <= 0)
    return JB_ERR_INVALID;
  // Tensor-core instantiation (3xTF32 wgmma for the three dense products): needs 128-row tiles (B % 128 == 0,
  // H % 128 == 0) and the W2 image workspaces.  It is parity-green but SLOWER than the FFMA tiles at the reference
  // minibatch (measured on H100 in DESIGN.md 8; the reason in DESIGN.md 3b: with 128-row tensor-core tiles only 32-64 CTAs work and each regenerates a 4x
  // larger operand panel on the CUDA cores, which is instruction-issue bound), so it is opt-in: JB_FUSED_TC=1.
  bool tc = false;
  if (const char* e = getenv("JB_FUSED_TC")) tc = atoi(e) != 0;
  tc = tc && a.B % 128 == 0 && a.H % 128 == 0 && a.W2img != nullptr && a.W2Timg != nullptr;
  int ctas = fused_max_ctas(a.B, tc, a.A, a.D);
  if (ctas <= 0) return JB_ERR_INVALID;
  if (ctas > NT) ctas = NT;
  if (a.world < 1 || a.world > 8 || a.rank < 0 || a.rank >= a.world) return JB_ERR_INVALID;
  if (a.world > 1) {   // grad must be this rank's exchange buffer: gradient | averaged gradient | flag words
    const long long q4 = (a.P4 + a.world - 1) / a.world;
    if (a.peer[a.rank] != a.grad || a.xllin_off < a.P4 * 4 || a.xgred_off < a.xllin_off + 8 * a.world * q4 ||
        a.xflag_off < a.xgred_off + 8 * a.P4 || (a.xllin_off & 7) || (a.xgred_off & 7) || (a.xflag_off & 3) || ctas > JB_X_MAX_CTAS)
      return JB_ERR_INVALID;
    for (int r = 0; r < a.world; ++r) if (!a.peer[r]) return JB_ERR_INVALID;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(a.barrier, 0, 64 * sizeof(unsigned int), s) != cudaSuccess) return JB_ERR_CUDA;   // grid counter, row-tile tickets, JB counters: monotonic targets from 0
  const size_t smem = fused_smem(a.B);
  int dsm_floats = dsm_floats_for(a.B);
  int flags = 0;
  if (const char* e = getenv("JB_FUSED_SKIP")) flags = atoi(e);     // bit 8: record the timing trace
  void* kargs[] = {&a, &dsm_floats, &flags};
  cudaError_t e = cudaLaunchCooperativeKernel(const_cast<void*>(fused_fn(tc, a.A, a.D)), dim3(ctas), dim3(NT), kargs, smem, s);
  if (e != cudaSuccess) { cudaGetLastError(); return JB_ERR_CUDA; }
  return JB_OK;
}
