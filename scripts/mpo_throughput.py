"""Throughput of MPO on one GPU, in one process, at the built-in configs' agent shapes (H=512, n=8, B=64, K=30):

  cartpole   config.mpo.cartpole (discrete, 2 actions), 8 actors
  mujoco     config.mpo.mujoco on the Hopper-shaped synthetic task (11-dim observation, 3 actions), 16 actors

Each case first collects through ReplayCollector (config update_period batched env steps per round, one learn() per
round, CUDA-graph learn) for `--warmup` rounds, then `--rounds` timed rounds; env-steps/s counts every actor's steps.
Then learn() alone is timed `--learns` times, alternating in blocks of 5 with SAC's learn() at the same shape (SAC's
config for the env with hidden_size 512 and batch_size 64 x n_step rows, the rows one MPO learn trains its critic on;
discrete SAC on CartPole), both on their CUDA graphs.  The GPU's name, power limit and SM clock come from a read-only
nvidia-smi query in the same run, taken after the cases.

  python scripts/mpo_throughput.py [--rounds 40] [--learns 50] [--warmup 10]
"""
import argparse
import contextlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402

CASES = {"cartpole": ("config.mpo.cartpole", "cartpole", "config.sac_discrete.cartpole"),
         "mujoco": ("config.mpo.mujoco", "hopper", "config.sac.mujoco")}


def _agent(cfg, env, **over):
    from jorldy_b200.core import Agent
    ag = dict(cfg.agent, start_train_step=0, lr_decay=False, **over)
    return Agent(**dict(ag, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
                        run_step=10 ** 9, device="cuda"))


def _fill(agent, env, N, rounds):
    from jorldy_b200.core.collect import ReplayCollector
    agent.start_train_step = 10 ** 9                 # collect only
    rc = ReplayCollector(env, agent, 32)
    step = 0
    for _ in range(rounds):
        step, _ = rc.run_round(step)
    agent.start_train_step = 0


def _time(agent, n):
    import torch
    out = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        agent.learn()                                   # ends in the host read of the stats: synchronised
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def run_case(name, rounds, learns, warmup):
    import numpy as np
    import torch
    from jorldy_b200 import config as cfgs
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    path, task, sac_path = CASES[name]
    cfg = cfgs.load(path)
    torch.cuda.reset_peak_memory_stats()
    N = int(cfg.train["num_workers"])
    update_period = int(cfg.train["update_period"])
    env_kw = {k: v for k, v in cfg.env.items() if k != "name"}
    env = Env(task, num_envs=N, seed=0, device="cuda", **env_kw)
    agent = _agent(cfg, env)
    rc = ReplayCollector(env, agent, update_period)
    step = 0
    for _ in range(warmup):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        step, res = rc.run_round(step)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    env_steps = rounds * update_period * N
    # SAC at the same shape: B * n rows per learn, H = 512
    scfg = cfgs.load(sac_path)
    senv = Env(task, num_envs=N, seed=1, device="cuda", **{k: v for k, v in scfg.env.items() if k != "name"})
    sac = _agent(scfg, senv, hidden_size=512, batch_size=agent.batch_size * agent.n_step)
    _fill(sac, senv, N, max(4, (agent.batch_size * agent.n_step) // (32 * N) + 2))
    for a in (agent, sac):
        _time(a, 3)                                     # warm: eager first learn, capture, replay
    mpo_ms, sac_ms = [], []
    for _ in range(max(1, learns // 5)):
        mpo_ms += _time(agent, 5)
        sac_ms += _time(sac, 5)
    med = lambda x: float(np.median(x))
    return {"case": name, "num_envs": N, "update_period": update_period, "batch_windows": agent.batch_size,
            "n_step": agent.n_step, "num_sample": agent.num_sample, "hidden": agent.actor.D_hidden,
            "collect_learn_env_steps_per_s": env_steps / dt, "timed_rounds": rounds,
            "mpo_learn_ms_median": med(mpo_ms), "mpo_learn_ms_min": min(mpo_ms),
            "sac_learn_ms_median": med(sac_ms), "sac_learn_ms_min": min(sac_ms), "sac_rows": sac.batch_size,
            "last_result": res, "peak_alloc_mb": torch.cuda.max_memory_allocated() / 2 ** 20}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cases", default="cartpole,mujoco")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mpo_throughput.py measures on a GPU; none is visible")
    with contextlib.redirect_stdout(sys.stderr):        # the replay's first-store report: stdout carries the JSON only
        cases = [run_case(c, args.rounds, args.learns, args.warmup) for c in args.cases.split(",")]
    print(json.dumps({"gpu": gpu_info(), "cases": cases}))


if __name__ == "__main__":
    main()
