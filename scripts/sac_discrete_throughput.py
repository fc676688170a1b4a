"""Throughput and memory of the discrete-action SAC on one GPU, in one process:

  cartpole_1024    discrete CartPole (config.sac_discrete.cartpole's agent, H=512), 1024 actors, B=64
  atari_16         config.sac_discrete.atari on synthetic seaquest frames (18 actions), 1M-slot single-frame replay, 16 lanes
  atari_256        the same behind 256 lanes

Each case collects through ReplayCollector with `--update-period` batched env steps per round and one learn() per round
(CUDA-graph learn), after `--warmup` rounds; env-steps/s counts every actor's steps over the timed rounds.  learn() alone
is then timed `--learns` times with the CUDA graph and `--learns` times eagerly (same agent, same replay), alternating in
blocks of 5.  Also printed: the peak allocation of the case and the GPU's name, power limit and SM clock (read-only
nvidia-smi query).

  python scripts/sac_discrete_throughput.py [--rounds 50] [--learns 50]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402

CASES = {"cartpole_1024": ("config.sac_discrete.cartpole", "cartpole", 1024, None),
         "atari_16": ("config.sac_discrete.atari", "seaquest", 16, 1_000_000),
         "atari_256": ("config.sac_discrete.atari", "seaquest", 256, 1_000_000)}


def _time_learns(agent, n, graph):
    import torch
    agent.use_cuda_graph = graph
    out = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        agent.learn()                                   # ends in the host read of the stats: synchronised
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def run_case(name, rounds, learns, update_period, warmup):
    import torch
    from jorldy_b200 import config as cfgs
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import ReplayCollector
    path, game, N, buffer_size = CASES[name]
    cfg = cfgs.load(path)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    env_kw = {k: v for k, v in cfg.env.items() if k != "name"}
    env = Env(game, num_envs=N, seed=0, device="cuda", **env_kw)
    ag = dict(cfg.agent, start_train_step=0, lr_decay=False)
    if buffer_size:
        ag["buffer_size"] = buffer_size
    agent = Agent(**dict(ag, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
                         run_step=10 ** 9, device="cuda"))
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
    tg, te = [], []
    for _ in range(max(1, learns // 5)):
        tg += _time_learns(agent, 5, True)
        te += _time_learns(agent, 5, False)
    agent.use_cuda_graph = True
    tg.sort(), te.sort()
    out = {"case": name, "config": path, "env": game, "actors": N, "actions": env.action_size, "batch_size": agent.batch_size,
           "hidden": agent.actor.D_hidden, "replay_slots": agent.memory.buffer_size, "update_period": update_period,
           "frame_store": agent.memory.frames is not None, "rounds": rounds,
           "env_steps_per_sec": N * update_period * rounds / dt, "ms_per_round": dt / rounds * 1e3,
           "ms_learn_graph_median": tg[len(tg) // 2], "ms_learn_graph_best": tg[0],
           "ms_learn_eager_median": te[len(te) // 2], "ms_learn_eager_best": te[0],
           "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(), "last_result": res}
    del rc, agent, env
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--update-period", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("sac_discrete_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    for name in args.cases.split(","):
        print(json.dumps(run_case(name, args.rounds, args.learns, args.update_period, args.warmup)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
