"""MuZero throughput on the GPU: env-steps/s and simulations/s of the batched search on CartPole, the act time per env
step from device events after warm-up, and the learn time at batch 128.  Each is timed over --steps (--learns) calls,
about a second of device time per window, and the three windows are repeated --repeats times in turn; the JSON line
gives every repeat and the median, with the card's name and power limit read in the same run.

    python scripts/muzero_throughput.py [--envs 256] [--sims 50] [--steps 500] [--learns 500] [--repeats 5]
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
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--sims", type=int, default=50)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--learns", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from jorldy_b200 import config as cfg
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import ReplayCollector
    a = dict(cfg.load("config.muzero.cartpole").agent, num_simulation=args.sims, start_train_step=10 ** 12)
    env = Env("cartpole", num_envs=args.envs, seed=0)
    agent = Agent(**a, state_size=4, action_size=2, run_step=10 ** 6, device="cuda")
    col = ReplayCollector(env, agent, update_period=1)
    for _ in range(agent.L + 2):                         # warm-up: graph capture and the first windows
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
        act.append(timed(lambda: agent.act_device(x, True), args.steps))      # the search alone
        rnd.append(timed(lambda: col.run_round(0), args.steps))               # act, env step, windows, replay store
        learn.append(timed(agent.learn, args.learns))                         # batch 128 from the filled replay
    med = lambda v: float(np.median(v))
    act_ms, round_ms, learn_ms = med(act), med(rnd), med(learn)
    print(json.dumps({"card": card(), "envs": args.envs, "num_simulation": args.sims, "act_ms_per_env_step": act_ms,
                      "round_ms_per_env_step": round_ms, "env_steps_per_s": args.envs / (round_ms / 1e3),
                      "simulations_per_s": args.envs * args.sims / (act_ms / 1e3), "learn_ms_b128": learn_ms,
                      "batch_size": agent.batch_size, "repeats": {"act_ms": act, "round_ms": rnd, "learn_ms": learn}}))


if __name__ == "__main__":
    main()
