"""MuZero on Atari frames, throughput on the GPU: `config.muzero.atari` on the synthetic Atari env (its 32 envs, S = 50,
batch 1024, the 1 M-window replay and its frame rings).  Reports the act time per env step (the search alone, from device
events), collection env-steps/s (act, env step, frame push, windows and the replay store) and the learn time, each over
--steps (--learns) calls after warm-up, repeated --repeats times in turn; and the peak device memory with the replay and
the frame rings allocated at the configured size.  One JSON line with every repeat, the medians and the card's name
and power limit, read in the same run.

    python scripts/muzero_frames_throughput.py [--envs 32] [--sims 50] [--steps 200] [--learns 50] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=32)
    ap.add_argument("--sims", type=int, default=50)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--buffer-size", type=int, default=None, help="windows (default: the config's)")
    args = ap.parse_args()
    from jorldy_b200 import config as cfg
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import ReplayCollector
    c = cfg.load("config.muzero.atari")
    a = dict(c.agent, num_simulation=args.sims, start_train_step=10 ** 12)
    if args.buffer_size:
        a["buffer_size"] = args.buffer_size
    env = Env("breakout", num_envs=args.envs, seed=0)
    agent = Agent(**a, state_size=env.state_size, action_size=env.action_size, optim_config=c.optim, run_step=10 ** 6,
                  device="cuda")
    col = ReplayCollector(env, agent, update_period=1)
    rounds = agent.L + max(2, -(-agent.batch_size // args.envs))     # graph capture, and a batch of windows
    for _ in range(rounds):
        col.run_round(0)
    torch.cuda.synchronize()
    x = env.obs.clone()
    agent.learn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    act, rnd, learn = [], [], []
    for _ in range(args.repeats):
        act.append(timed(lambda: agent.act_device(x, True), args.steps))
        rnd.append(timed(lambda: col.run_round(0), args.steps))
        learn.append(timed(agent.learn, args.learns))
    med = lambda v: float(np.median(v))
    act_ms, round_ms, learn_ms = med(act), med(rnd), med(learn)
    print(json.dumps({"card": card(), "envs": args.envs, "num_simulation": args.sims, "batch_size": agent.batch_size,
                      "buffer_size": agent.buffer_size, "frames_per_lane": agent._frames.F,
                      "act_ms_per_env_step": act_ms, "round_ms_per_env_step": round_ms,
                      "env_steps_per_s": args.envs / (round_ms / 1e3), "learn_ms": learn_ms,
                      "peak_memory_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
                      "repeats": {"act_ms": act, "round_ms": rnd, "learn_ms": learn}}))


if __name__ == "__main__":
    main()
