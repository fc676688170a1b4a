// Single-frame Atari replay: every 84x84 frame is stored once, in a per-lane ring, and a replay slot holds two int64 frame
// references instead of two [4,84,84] stacks (jorldy_b200/core/buffer/frame_store.py owns the format).
//
// Layout, per lane (one batched env row) e of n:
//   frames[e][F][7056]  uint8, frame of absolute position p at slot p % F
//   first[e][F]         int64, absolute position of the episode-first frame of the frame at that slot
//   head[e]             int64, number of frames pushed so far (the next absolute position)
// A reference is (e << 40) | p.  The stack at position p is frames[max(p - 3 + k, first[p])] for k = 0..3: the newest
// frame last, and the episode-first frame repeated where the episode is shorter than the stack — exactly the reset
// observation (first frame tiled x4, csrc/env_frames.cu) and every shifted stack after it.
//
// Push (one CTA per lane, 441 uint4 per frame): the newest frame of next_obs continues the episode of the stack acted
// on; when the env auto-reset, obs[:,3] (the new first frame) follows as an episode-first frame.  Writes 1-2 frames
// = 7-14 KB per lane and step, against 56 KB of stacks in the duplicated layout; HBM-write-bound at large n.
// Gather (grid = sample x {state, next} x stack slot, one contiguous 7056-byte frame per CTA): a reference whose frames
// are no longer resident (an overwritten slot) is never read: its output is zeroed and *status is set, for the host to
// raise on.  At B = 32..512 the gather moves 0.9..14 MB and is launch-latency-bound.
// PPO's frame rollout keeps its states on the same rings; im2col_u8_frames_kernel below writes conv1's column matrix
// straight from them, with the gather's stack rule and residency check, and with MuZero's action planes appended.
#include "common.cuh"

namespace {

constexpr int FRAME = 84 * 84;          // 7056 bytes = 441 uint4
constexpr int FRAME_VEC = FRAME / 16;
constexpr int STACK = 4;
constexpr int POS_BITS = 40;
constexpr long long POS_MASK = (1LL << POS_BITS) - 1;

__device__ __forceinline__ void copy_frame(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src) {
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (int q = threadIdx.x; q < FRAME_VEC; q += blockDim.x) d[q] = s[q];
}

__global__ void frame_push_kernel(uint8_t* __restrict__ frames, int64_t* __restrict__ first, int64_t* __restrict__ head,
                                  long long F, const uint8_t* __restrict__ obs, const uint8_t* __restrict__ next_obs,
                                  const float* __restrict__ done, int auto_reset, int64_t* __restrict__ state_ref,
                                  int64_t* __restrict__ next_ref) {
  const long long e = blockIdx.x;
  uint8_t* ring = frames + (size_t)e * F * FRAME;
  int64_t* fst = first + e * F;
  long long h = head[e];
  bool reset = true;
  if (next_obs) {
    const long long cont = fst[(h - 1) % F];          // episode of the stack acted on (position h - 1)
    copy_frame(ring + (size_t)(h % F) * FRAME, next_obs + ((size_t)e * STACK + 3) * FRAME);
    if (threadIdx.x == 0) {
      fst[h % F] = cont;
      if (state_ref) state_ref[e] = (e << POS_BITS) | (h - 1);
      if (next_ref) next_ref[e] = (e << POS_BITS) | h;
    }
    h += 1;
    reset = auto_reset && done[e] > 0.5f;
  }
  if (reset) {
    copy_frame(ring + (size_t)(h % F) * FRAME, obs + ((size_t)e * STACK + 3) * FRAME);
    if (threadIdx.x == 0) fst[h % F] = h;
    h += 1;
  }
  __syncthreads();                                   // every thread has read head[e] before it moves
  if (threadIdx.x == 0) head[e] = h;
}

__global__ void frame_gather_kernel(const uint8_t* __restrict__ frames, const int64_t* __restrict__ first,
                                    const int64_t* __restrict__ head, long long F, int n_lanes,
                                    const int64_t* __restrict__ state_refs, const int64_t* __restrict__ next_refs,
                                    const int64_t* __restrict__ idx, uint8_t* __restrict__ state_out,
                                    uint8_t* __restrict__ next_out, int32_t* __restrict__ status) {
  const long long b = blockIdx.x;
  const int which = blockIdx.y, k = blockIdx.z;
  const int64_t* refs = which ? next_refs : state_refs;
  const long long r = refs[idx ? idx[b] : b];
  uint8_t* dst = (which ? next_out : state_out) + ((size_t)b * STACK + k) * FRAME;
  const long long lane = r >> POS_BITS, p = r & POS_MASK;
  bool ok = r >= 0 && lane < n_lanes;
  long long src = 0;
  if (ok) {
    const long long h = head[lane];
    ok = p < h && p >= h - F;                        // the slot of p still holds p, so first[] below is p's
    if (ok) {
      const long long f = first[lane * F + p % F];
      const long long lo = p - 3 > f ? p - 3 : f;    // oldest frame of the stack
      ok = lo >= h - F && f <= p;
      const long long q = p - 3 + k > f ? p - 3 + k : f;
      src = lane * F + q % F;
    }
  }
  if (ok) {
    copy_frame(dst, frames + (size_t)src * FRAME);
  } else {
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (int q = threadIdx.x; q < FRAME_VEC; q += blockDim.x) d[q] = make_uint4(0, 0, 0, 0);
    if (threadIdx.x == 0) *reinterpret_cast<volatile int32_t*>(status) = 1;
  }
}

// conv1's im2col (8x8 kernel, stride 4, 4x84x84 -> 20x20 outputs, K = 256 in im2col_u8_nchw_vec4_kernel's order
// c*64 + ky*8 + kx) read straight from the ring: grid = (stack i, output row oy), 256 threads.  Four threads resolve the
// stack's four source frames (the stack rule and residency check of frame_gather_kernel) into shared memory; then each
// thread turns one 4-byte frame-row load into one 16-byte column store, five times: 20 x 64 float4 = 20 KB per CTA.
// PLANES (MuZero's representation input): four more channels c = 4 + k, each the constant a_k / A, where a_k
// (actions[row][k]) is the action that produced stack frame k; a frame at or before its episode's first frame was
// produced by no action and gets an all-zero plane.  K = 512, ten column stores per thread, 40 KB per CTA.
constexpr int OUT = 20, KSZ = 8, STRIDE = 4;

template <bool PLANES>
__global__ void __launch_bounds__(256) im2col_u8_frames_kernel(
    const uint8_t* __restrict__ frames, const int64_t* __restrict__ first, const int64_t* __restrict__ head, long long F,
    int n_lanes, const int64_t* __restrict__ refs, const int32_t* __restrict__ idx, const int64_t* __restrict__ actions,
    int num_actions, float* __restrict__ col, int32_t* __restrict__ status) {
  constexpr int K4 = (PLANES ? 2 : 1) * STACK * KSZ * KSZ / 4;
  constexpr int ROW_VEC = OUT * K4;              // float4 of one output row oy of one stack
  __shared__ long long src[STACK];               // frame index lane * F + slot, or -1 when the stack is not resident
  __shared__ float plane[STACK];
  const long long i = blockIdx.x;
  const int oy = blockIdx.y;
  if (threadIdx.x < STACK) {
    const int k = threadIdx.x;
    const long long row = idx ? idx[i] : i;
    const long long r = refs[row];
    const long long lane = r >> POS_BITS, p = r & POS_MASK;
    bool ok = r >= 0 && lane < n_lanes;
    long long s = -1;
    float a = 0.f;
    if (ok) {
      const long long h = head[lane];
      ok = p < h && p >= h - F;
      if (ok) {
        const long long f = first[lane * F + p % F];
        const long long lo = p - 3 > f ? p - 3 : f;
        ok = lo >= h - F && f <= p;
        const long long q = p - 3 + k > f ? p - 3 + k : f;
        s = ok ? lane * F + q % F : -1;
        if (PLANES && ok && p - 3 + k > f) a = __fdiv_rn((float)actions[row * STACK + k], (float)num_actions);
      }
    }
    src[k] = s;
    if (PLANES) plane[k] = a;
    if (!ok && k == 0 && oy == 0) *reinterpret_cast<volatile int32_t*>(status) = 1;
  }
  __syncthreads();
  float4* out = reinterpret_cast<float4*>(col) + ((size_t)i * OUT + oy) * ROW_VEC;
  for (int q = threadIdx.x; q < ROW_VEC; q += blockDim.x) {
    const int ox = q / K4, k4 = q % K4;
    const int kx4 = k4 & 1, ky = (k4 >> 1) & (KSZ - 1), c = k4 >> 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (PLANES && c >= STACK) {
      const float a = plane[c - STACK];
      v = make_float4(a, a, a, a);
    } else {
      const long long s = src[c];
      if (s >= 0) {
        const uchar4 u = *reinterpret_cast<const uchar4*>(frames + (size_t)s * FRAME + (oy * STRIDE + ky) * 84 +
                                                           ox * STRIDE + 4 * kx4);
        v = make_float4((float)u.x / 255.0f, (float)u.y / 255.0f, (float)u.z / 255.0f, (float)u.w / 255.0f);
      }
    }
    out[q] = v;
  }
}

}  // namespace

JB_API int jb_frame_push(uint8_t* frames, int64_t* first, int64_t* head, int64_t frames_per_lane, const uint8_t* obs,
                         const uint8_t* next_obs, const float* done, int auto_reset, int64_t* state_ref, int64_t* next_ref,
                         int n, void* stream) {
  if (!frames || !first || !head || !obs || n <= 0 || frames_per_lane < 8 || (next_obs && !done)) return JB_ERR_INVALID;
  frame_push_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(frames, first, head, frames_per_lane, obs, next_obs, done,
                                                         auto_reset, state_ref, next_ref);
  return jb_check_launch();
}

JB_API int jb_frame_gather(const uint8_t* frames, const int64_t* first, const int64_t* head, int64_t frames_per_lane,
                           int n_lanes, const int64_t* state_refs, const int64_t* next_refs, const int64_t* idx, int B,
                           uint8_t* state_out, uint8_t* next_out, int32_t* status, void* stream) {
  if (!frames || !first || !head || !state_refs || !next_refs || !state_out || !next_out || !status || B <= 0 ||
      n_lanes <= 0 || frames_per_lane < 8)
    return JB_ERR_INVALID;
  frame_gather_kernel<<<dim3(B, 2, STACK), 128, 0, (cudaStream_t)stream>>>(frames, first, head, frames_per_lane, n_lanes,
                                                                            state_refs, next_refs, idx, state_out, next_out,
                                                                            status);
  return jb_check_launch();
}

JB_API int jb_im2col_u8_frames(const uint8_t* frames, const int64_t* first, const int64_t* head, int64_t frames_per_lane,
                               int n_lanes, const int64_t* refs, const int32_t* idx, int M, float* col, int32_t* status,
                               void* stream) {
  if (!frames || !first || !head || !refs || !col || !status || M <= 0 || n_lanes <= 0 ||
      frames_per_lane < 8 || (((uintptr_t)frames & 3) | ((uintptr_t)col & 15)))
    return JB_ERR_INVALID;
  im2col_u8_frames_kernel<false><<<dim3(M, OUT), 256, 0, (cudaStream_t)stream>>>(
      frames, first, head, frames_per_lane, n_lanes, refs, idx, nullptr, 0, col, status);
  return jb_check_launch();
}

JB_API int jb_im2col_u8_frames_actions(const uint8_t* frames, const int64_t* first, const int64_t* head,
                                       int64_t frames_per_lane, int n_lanes, const int64_t* refs, const int64_t* actions,
                                       int num_actions, const int32_t* idx, int M, float* col, int32_t* status,
                                       void* stream) {
  if (!frames || !first || !head || !refs || !actions || !col || !status || M <= 0 || n_lanes <= 0 ||
      num_actions <= 0 || frames_per_lane < 8 || (((uintptr_t)frames & 3) | ((uintptr_t)col & 15)))
    return JB_ERR_INVALID;
  im2col_u8_frames_kernel<true><<<dim3(M, OUT), 256, 0, (cudaStream_t)stream>>>(
      frames, first, head, frames_per_lane, n_lanes, refs, idx, actions, num_actions, col, status);
  return jb_check_launch();
}
