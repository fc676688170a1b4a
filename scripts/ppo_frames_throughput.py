"""Throughput and memory of PPO on Atari frames (FrameRollout: states kept as single-frame references, conv1's im2col
read from the frame ring), on one GPU, in one process:

  reference   config.ppo.atari at the reference's scale: 8 envs, T=128, B=256 (distributed_batch_size), 3 epochs, H=512, on
              --game (default breakout, A=4; seaquest has ALE's full 18 actions)
  scaled      the same with 1024 envs

Each configuration runs one collect() + learn_rollout() as warm-up (CUDA-graph capture), then times three repeats of
collect() and learn_rollout() with CUDA events, and reports the best and the spread.  A comparison at 256 envs times
learn_rollout() on the frame rollout and _learn_tensors() on the same rollout materialised as uint8 [N*T,4,84,84] stacks,
alternating 3x.  Also printed: the rollout's bytes per env (arithmetic) and the GPU's name, power limit and SM clock
(read-only nvidia-smi query).

  python scripts/ppo_frames_throughput.py [--repeats 3] [--game breakout]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402

T, B, EPOCHS, H = 128, 256, 3, 512
GAME = "breakout"
FRAME = 84 * 84


def rollout_bytes_per_env(T):
    """HBM per env: the ring's frames and episode-first positions, its head, and per step a state reference, an int32
    action, reward and done, plus the last next-state reference."""
    from jorldy_b200.core.buffer.frame_store import frames_per_rollout
    F = frames_per_rollout(T)
    return {"frame_rollout": F * (FRAME + 8) + 8 + T * (8 + 4 + 4 + 4) + 8,
            "uint8_stacks": (T + 1) * 4 * FRAME + T * 12, "fp32_stacks": (T + 1) * 4 * FRAME * 4 + T * 12,
            "ring_frames": F, "ring_frame_bytes": F * FRAME}


def _agent(n_step=T):
    from jorldy_b200.core import Agent
    from jorldy_b200.core.env.frames import _ACTIONS
    return Agent("ppo", state_size=[4, 84, 84], action_size=_ACTIONS[GAME], hidden_size=H, head="cnn", n_step=n_step,
                 batch_size=B, n_epoch=EPOCHS, optim_config={"name": "adam", "lr": 2.5e-4}, run_step=10 ** 9,
                 lr_decay=False, device="cuda")


def _timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def run_config(name, N, repeats):
    import torch
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    agent = _agent()
    col = RolloutCollector(Env(GAME, num_envs=N, seed=0, device="cuda"), agent)
    agent.learn_rollout(col.collect())                  # warm-up: graph capture of collect and of the minibatch chunk
    torch.cuda.synchronize()
    tc, tl = [], []
    for _ in range(repeats):
        c_ms, ro = _timed(col.collect)
        l_ms, _ = _timed(lambda: agent.learn_rollout(ro))
        tc.append(c_ms)
        tl.append(l_ms)
    tot = [c + l for c, l in zip(tc, tl)]
    out = {"config": name, "envs": N, "T": T, "batch_size": B, "n_epoch": EPOCHS, "hidden": H, "game": GAME,
           "actions": agent.action_size,
           "env_steps_per_sec": N * T / (min(tot) / 1e3),
           "learner_transitions_per_sec": N * T * EPOCHS / (min(tl) / 1e3),
           "ms_collect_best": min(tc), "ms_collect_spread": max(tc) - min(tc),
           "ms_learn_best": min(tl), "ms_learn_spread": max(tl) - min(tl),
           "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(),
           "rollout_bytes_per_env": rollout_bytes_per_env(T)["frame_rollout"], "status_word": int(col.rollout.frames.status[0])}
    del col, agent
    torch.cuda.empty_cache()
    return out


def compare(N, repeats):
    """learn_rollout() on the frame rollout vs _learn_tensors() on its materialised uint8 stacks, alternating."""
    import torch
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    torch.cuda.empty_cache()
    a, b = _agent(), _agent()
    b.network.load_state_dict(a.network.state_dict())
    ro = RolloutCollector(Env(GAME, num_envs=N, seed=0, device="cuda"), a).collect()
    refs = ro.state_ref.reshape(-1)
    stacks, _ = ro.frames.gather(refs, refs)
    last, _ = ro.frames.gather(ro.last_next_state, ro.last_next_state)
    args = (ro.action.reshape(-1), ro.reward.reshape(-1), ro.done.reshape(-1))

    def frames():
        return a.learn_rollout(ro)

    def stacked():
        return b._learn_tensors(stacks, *args, last_next_state=last)

    frames()                                            # warm-up both (graph capture)
    stacked()
    tf, ts = [], []
    for _ in range(repeats):
        tf.append(_timed(frames)[0])
        ts.append(_timed(stacked)[0])
    out = {"compare_envs": N, "ms_learn_frames": tf, "ms_learn_uint8_stacks": ts,
           "frames_best_ms": min(tf), "stacks_best_ms": min(ts), "frames_faster": min(tf) < min(ts)}
    del a, b, ro, stacks
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scaled-envs", type=int, default=1024)
    ap.add_argument("--compare-envs", type=int, default=256)
    ap.add_argument("--game", type=str, default="breakout")
    args = ap.parse_args()
    global GAME
    GAME = args.game
    import torch
    if not torch.cuda.is_available():
        sys.exit("ppo_frames_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info(), "bytes_per_env": rollout_bytes_per_env(T)}),
          flush=True)
    print(json.dumps(run_config("reference", 8, args.repeats)), flush=True)
    print(json.dumps(run_config("scaled", args.scaled_envs, args.repeats)), flush=True)
    print(json.dumps(compare(args.compare_envs, args.repeats)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
