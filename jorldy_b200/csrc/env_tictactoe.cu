// Batched TicTacToe: one thread per board, against a uniform-random opponent (RANDOM), against a perfect player
// (PERFECT), or in self-play (SELF).
//
// The reference's tictactoe env source is not available, so these rules are this project's (DESIGN.md 5i, "MuZero on
// TicTacToe"):
//   - boards int32 [n, 2]: bit c of boards[i, 0] is the agent's mark on cell c (row-major 3x3), of boards[i, 1] the
//     opponent's;
//   - obs f32 [n, 18]: cells 0..8 = the agent's marks, 9..17 = the opponent's; legal u8 [n, 9] = the empty cells of obs;
//   - reset: an empty board; one Philox draw decides (u < 1/2) whether the opponent opens, on cell floor(u' 9);
//   - step(a): an occupied cell or an a outside 0..8 forfeits (-1, done, board unchanged); else the agent's mark, +1 and done
//     on a line, 0 and done on a full board; else the opponent's mark on the k-th empty cell, k = floor(u n_empty),
//     -1 and done on its line, 0 and done on a full board; else 0.
// Draws come from the env's own Philox stream (stream_base | env) at counter (episode << 4) | move, move 0 the opening
// and move m the reply to the agent's m-th move, so every episode and every replay of a captured collect draws fresh
// numbers.  Every game ends within the agent's 5th move.
//
// PERFECT: as RANDOM, but the opponent's cell is the k-th set bit of best[position] (k = floor(u popcount), u the draw
// RANDOM uses at the same counter), best u16 [3^9] the moves that reach the negamax value (core/env/tictactoe.py
// solve()), indexed in base 3 from the side to move: digit c is 1 for its mark on cell c, 2 for the other side's.  At the
// empty board every cell is optimal, so the opening is RANDOM's and PERFECT resets with RANDOM's kernel.  A board
// stepped after its game ended (without auto-reset) is outside the table (0 there); the opponent then takes any empty
// cell, as RANDOM does.
//
// SELF (two-player self-play): boards[i] = (side to move, other side) and obs in that order, so the mover always sees
// the board as the agent does above.  reset: an empty board, no draw.  step(a): an occupied cell or an a outside 0..8
// forfeits (-1 to the mover, done); a line +1, done; a full board 0, done; else 0.  After any move the sides swap, so
// next_obs is the board seen by the side that did not just move, at done too.  elapsed counts plies (at most 9) and
// score is the first player's outcome.
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int FULL = 0x1ff;
enum Opponent { RANDOM = 0, PERFECT = 1, SELF = 2 };

__device__ __forceinline__ bool has_line(int b) {
  const int lines[8] = {0x007, 0x038, 0x1c0, 0x049, 0x092, 0x124, 0x111, 0x054};
  bool w = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) w |= (b & lines[k]) == lines[k];
  return w;
}

// the k-th (0-based) set bit of m, ascending
__device__ __forceinline__ int kth_bit(int m, int k) {
  for (int j = 0; j < k; ++j) m &= m - 1;
  return __ffs(m) - 1;
}

__device__ __forceinline__ jb_philox4 draw(uint64_t seed, uint64_t stream_base, int i, int64_t episode, int move) {
  return jb_philox(seed, stream_base | (uint64_t)i, ((uint64_t)episode << 4) | (uint64_t)move);
}

__device__ __forceinline__ void write_board(int me, int op, float* __restrict__ obs, uint8_t* __restrict__ legal, int i) {
#pragma unroll
  for (int c = 0; c < 9; ++c) {
    obs[18 * i + c] = (float)((me >> c) & 1);
    obs[18 * i + 9 + c] = (float)((op >> c) & 1);
    if (legal) legal[9 * i + c] = (uint8_t)((((me | op) >> c) & 1) ^ 1);
  }
}

// base-3 index of a position from the side to move: digit c is 1 for the mover's mark on cell c, 2 for the other's
__device__ __forceinline__ int position(int mover, int other) {
  int idx = 0;
#pragma unroll
  for (int c = 8; c >= 0; --c) idx = 3 * idx + ((mover >> c) & 1) + 2 * ((other >> c) & 1);
  return idx;
}

// a new episode: episode + 1; against an opponent it opens with probability 1/2, in self-play the board stays empty
template <int OPP>
__device__ __forceinline__ void new_game(int& me, int& op, int64_t& ep, uint64_t seed, uint64_t stream_base, int i) {
  ep += 1;
  if (OPP == SELF) {
    me = 0;
    op = 0;
    return;
  }
  const jb_philox4 r = draw(seed, stream_base, i, ep, 0);
  me = 0;
  op = 0;
  if (jb_u01_double(r.x, r.y) < 0.5) op = 1 << min((int)(jb_u01_double(r.z, r.w) * 9.0), 8);
}

template <int OPP>
__global__ void ttt_reset_kernel(int32_t* __restrict__ boards, float* __restrict__ obs, uint8_t* __restrict__ legal,
                                 int32_t* __restrict__ elapsed, int64_t* __restrict__ episode,
                                 float* __restrict__ score, const uint8_t* __restrict__ mask, uint64_t seed,
                                 uint64_t stream_base, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (mask && !mask[i])) return;
  int me, op;
  int64_t ep = episode[i];
  new_game<OPP>(me, op, ep, seed, stream_base, i);
  episode[i] = ep;
  boards[2 * i] = me;
  boards[2 * i + 1] = op;
  write_board(me, op, obs, legal, i);
  elapsed[i] = 0;
  score[i] = 0.f;
}

template <int OPP>
__global__ void ttt_step_kernel(int32_t* __restrict__ boards, float* __restrict__ obs, uint8_t* __restrict__ legal,
                                int32_t* __restrict__ elapsed, int64_t* __restrict__ episode,
                                float* __restrict__ score, const void* __restrict__ action, int action_kind,
                                float* __restrict__ next_obs, float* __restrict__ reward, float* __restrict__ done,
                                float* __restrict__ stats, int auto_reset, uint64_t seed, uint64_t stream_base, int n,
                                const uint16_t* __restrict__ best) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int me = boards[2 * i], op = boards[2 * i + 1];
  int64_t ep = episode[i];
  const long long a = action_kind == 0 ? (long long)((const int64_t*)action)[i] : (long long)((const int32_t*)action)[i];
  const int el = elapsed[i] + 1;
  float r = 0.f;
  bool d = true;
  if (a < 0 || a > 8 || ((me | op) >> a) & 1) {
    r = -1.f;                                            // forfeit
  } else {
    me |= 1 << a;
    if (has_line(me)) r = 1.f;
    else if (OPP == SELF) d = (me | op) == FULL;
    else if ((me | op) != FULL) {
      int cells = FULL & ~(me | op);
      if (OPP == PERFECT) {          // a board stepped after its game ended is outside the table: any empty cell
        const int optimal = best[position(op, me)];
        if (optimal) cells = optimal;
      }
      const jb_philox4 q = draw(seed, stream_base, i, ep, el);
      const int k = min((int)(jb_u01_double(q.x, q.y) * (double)__popc(cells)), __popc(cells) - 1);
      op |= 1 << kth_bit(cells, k);
      if (has_line(op)) r = -1.f;
      else d = (me | op) == FULL;
    }
  }
  float sc = score[i] + r;
  if (OPP == SELF) {                 // the first player's outcome; then the other side moves next
    if (!(el & 1)) sc = score[i] - r;
    const int t = me;
    me = op;
    op = t;
  }
  write_board(me, op, next_obs, nullptr, i);
  reward[i] = r;
  done[i] = d ? 1.f : 0.f;
  int el_out = el;
  float sc_out = sc;
  if (d && auto_reset) {
    if (stats) { atomicAdd(&stats[0], 1.0f); atomicAdd(&stats[1], sc); }    // integer-valued: any order is exact
    new_game<OPP>(me, op, ep, seed, stream_base, i);
    episode[i] = ep;
    el_out = 0;
    sc_out = 0.f;
  }
  boards[2 * i] = me;
  boards[2 * i + 1] = op;
  write_board(me, op, obs, legal, i);
  elapsed[i] = el_out;
  score[i] = sc_out;
}

}  // namespace

JB_API int jb_env_tictactoe_reset(int32_t* boards, float* obs, uint8_t* legal, int32_t* elapsed, int64_t* episode,
                                  float* score, const uint8_t* mask, uint64_t seed, uint64_t stream_base, int n,
                                  void* stream) {
  if (n <= 0 || !boards || !obs || !legal || !elapsed || !episode || !score) return JB_ERR_INVALID;
  const int threads = 128;
  ttt_reset_kernel<RANDOM><<<jb_div_up(n, threads), threads, 0, (cudaStream_t)stream>>>(
      boards, obs, legal, elapsed, episode, score, mask, seed, stream_base, n);
  return jb_check_launch();
}

JB_API int jb_env_tictactoe_step(int32_t* boards, float* obs, uint8_t* legal, int32_t* elapsed, int64_t* episode,
                                 float* score, const void* action, int action_kind, float* next_obs, float* reward,
                                 float* done, float* stats, int auto_reset, uint64_t seed, uint64_t stream_base, int n,
                                 void* stream) {
  if (n <= 0 || !boards || !obs || !legal || !elapsed || !episode || !score || !action || !next_obs || !reward ||
      !done || (action_kind != 0 && action_kind != 1))
    return JB_ERR_INVALID;
  const int threads = 128;
  ttt_step_kernel<RANDOM><<<jb_div_up(n, threads), threads, 0, (cudaStream_t)stream>>>(
      boards, obs, legal, elapsed, episode, score, action, action_kind, next_obs, reward, done, stats, auto_reset, seed,
      stream_base, n, nullptr);
  return jb_check_launch();
}

namespace {

// the table goes with PERFECT and only with it
bool opponent_ok(int opponent, const uint16_t* best) {
  return (opponent == RANDOM || opponent == PERFECT || opponent == SELF) && (opponent == PERFECT) == (best != nullptr);
}

}  // namespace

JB_API int jb_env_tictactoe_reset_opp(int opponent, const uint16_t* best, int32_t* boards, float* obs, uint8_t* legal,
                                      int32_t* elapsed, int64_t* episode, float* score, const uint8_t* mask,
                                      uint64_t seed, uint64_t stream_base, int n, void* stream) {
  if (n <= 0 || !boards || !obs || !legal || !elapsed || !episode || !score || !opponent_ok(opponent, best))
    return JB_ERR_INVALID;
  const int threads = 128;
  const dim3 grid(jb_div_up(n, threads));
  cudaStream_t s = (cudaStream_t)stream;
  if (opponent == SELF)
    ttt_reset_kernel<SELF><<<grid, threads, 0, s>>>(boards, obs, legal, elapsed, episode, score, mask, seed,
                                                    stream_base, n);
  else                               // PERFECT opens like RANDOM: every cell of the empty board is optimal
    ttt_reset_kernel<RANDOM><<<grid, threads, 0, s>>>(boards, obs, legal, elapsed, episode, score, mask, seed,
                                                      stream_base, n);
  return jb_check_launch();
}

JB_API int jb_env_tictactoe_step_opp(int opponent, const uint16_t* best, int32_t* boards, float* obs, uint8_t* legal,
                                     int32_t* elapsed, int64_t* episode, float* score, const void* action,
                                     int action_kind, float* next_obs, float* reward, float* done, float* stats,
                                     int auto_reset, uint64_t seed, uint64_t stream_base, int n, void* stream) {
  if (n <= 0 || !boards || !obs || !legal || !elapsed || !episode || !score || !action || !next_obs || !reward ||
      !done || (action_kind != 0 && action_kind != 1) || !opponent_ok(opponent, best))
    return JB_ERR_INVALID;
  const int threads = 128;
  const dim3 grid(jb_div_up(n, threads));
  cudaStream_t s = (cudaStream_t)stream;
  if (opponent == RANDOM)
    ttt_step_kernel<RANDOM><<<grid, threads, 0, s>>>(boards, obs, legal, elapsed, episode, score, action, action_kind,
                                                     next_obs, reward, done, stats, auto_reset, seed, stream_base, n,
                                                     best);
  else if (opponent == PERFECT)
    ttt_step_kernel<PERFECT><<<grid, threads, 0, s>>>(boards, obs, legal, elapsed, episode, score, action, action_kind,
                                                      next_obs, reward, done, stats, auto_reset, seed, stream_base, n,
                                                      best);
  else
    ttt_step_kernel<SELF><<<grid, threads, 0, s>>>(boards, obs, legal, elapsed, episode, score, action, action_kind,
                                                   next_obs, reward, done, stats, auto_reset, seed, stream_base, n,
                                                   best);
  return jb_check_launch();
}
