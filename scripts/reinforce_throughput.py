"""REINFORCE collect + learn throughput on one GPU, in one process; prints one JSON document.

  cartpole  config.reinforce.cartpole's sizes at 4096 CartPole envs (T_round = 128, H = 512, discrete_policy)
  hopper    config.reinforce.mujoco's sizes at Hopper dimensions (32 envs, T_round = 2048, H = 512, continuous_policy)

For each: env steps/s of collect + learn, collect and learn ms per round, the M of each learn, learn ms per chunk, the
launches per learn, and the per-round mean score (episodes finished in the round) as a learning-curve sanity check.
The first round (collect-graph capture and chunk-graph capture) is not timed.
gpu: name, power limit and SM clock (read-only nvidia-smi query), read before and after.

  python scripts/reinforce_throughput.py [--rounds 8]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402
from ppo_frames_throughput import _timed  # noqa: E402

CASES = {
    "cartpole": dict(config="config.reinforce.cartpole", env="cartpole", N=4096),
    "hopper": dict(config="config.reinforce.mujoco", env="hopper", N=32),
}


def run_case(name, rounds):
    import torch
    from jorldy_b200 import config as cfgs
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import EpisodeCollector
    s = CASES[name]
    cfg = cfgs.load(s["config"])
    T = int(cfg.train["update_period"])
    env = Env(s["env"], num_envs=s["N"], seed=0, device="cuda")
    agent = Agent(**dict(cfg.agent, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
                         run_step=10 ** 9, lr_decay=False, device="cuda"))
    col = EpisodeCollector(env, agent, T)
    agent.learn_episodes(col.collect())              # graph captures
    torch.cuda.synchronize()
    env.stats.zero_()
    per_round = []
    for _ in range(rounds):
        c_ms, ring = _timed(col.collect)
        l_ms, res = _timed(lambda: agent.learn_episodes(ring))
        ep, sc = env.stats.tolist()
        env.stats.zero_()
        n_chunks = -(-agent.last_M // agent._chunk_rows(ring))
        per_round.append({"collect_ms": c_ms, "learn_ms": l_ms, "M": agent.last_M, "chunks": n_chunks,
                          "learn_ms_per_chunk": l_ms / n_chunks if n_chunks else None, "launches": agent.n_launches,
                          "episodes": int(ep), "mean_score": sc / ep if ep else None, "loss": res.get("loss")})
    sps = [s["N"] * T / ((r["collect_ms"] + r["learn_ms"]) / 1e3) for r in per_round]
    return {"case": name, "config": s["config"], "envs": s["N"], "T_round": T, "hidden_size": agent.network.D_hidden,
            "ring_L": col.ring.L, "chunk_rows": agent._chunk_rows(col.ring), "env_steps_per_sec_best": max(sps),
            "env_steps_per_sec": sps, "rounds": per_round}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("reinforce_throughput.py measures on a CUDA device; none is available")
    doc = {"gpu": torch.cuda.get_device_name(0), "gpu_before": gpu_info()}
    doc["cases"] = [run_case(k, args.rounds) for k in CASES]
    doc["gpu_after"] = gpu_info()
    print(json.dumps(doc), flush=True)


if __name__ == "__main__":
    main()
