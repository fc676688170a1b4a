"""RND-PPO against ICM-PPO and PPO's multi-launch path on one GPU, in one process; prints one JSON document.

  learn   learn_rollout() ms of RND-PPO, ICM-PPO and PPO with use_fused=False (the CUDA-graph multi-launch path both share)
          on the same collected rollout, alternated for --repeats rounds, at the ppo_cartpole benchmark shape (4096
          CartPole envs, T = 128, B = 256, 3 epochs, H = 512) and at Hopper dimensions with config.ppo.mujoco's sizes
          (32 envs, T = 2048, B = 512, 10 epochs, H = 512); launches per minibatch and peak memory of each
  kernels jb_rnd_ppo_loss against jb_ppo_loss (each with its finalize) and jb_rnd_loss at B = 256 / 2048, CUDA events
          over 100 launches
  frames  collect + learn env steps/s of RND-PPO on synthetic Atari frames (CNN head and CNN RND, A = 18, T = 128,
          B = 256, 3 epochs, H = 512) at 8 and 256 envs, and peak memory
  gpu     name, power limit and SM clock (read-only nvidia-smi query), read before and after

  python scripts/rnd_ppo_throughput.py [--repeats 3] [--out PATH]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402
from icm_ppo_throughput import LEARN_SHAPES, _events  # noqa: E402
from ppo_frames_throughput import _timed  # noqa: E402


def learn_case(name, repeats):
    import torch
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    s = LEARN_SHAPES[name]
    env = Env(s["env"], num_envs=s["N"], seed=0, device="cuda")
    mk = lambda algo, **kw: Agent(algo, state_size=env.state_size, action_size=env.action_size, hidden_size=512,
                                  network=s["net"], n_step=s["T"], batch_size=s["B"], n_epoch=s["epochs"],
                                  optim_config={"name": "adam", "lr": s["lr"]}, run_step=10 ** 9, lr_decay=False,
                                  device="cuda", **kw)
    agents = {"rnd_ppo": mk("rnd_ppo"), "icm_ppo": mk("icm_ppo"), "ppo_multilaunch": mk("ppo", use_fused=False)}
    ro = RolloutCollector(env, agents["rnd_ppo"]).collect()      # keeps next_state; PPO reads only what it always did
    T = s["T"]
    for a in agents.values():                         # warm-up: graph capture, workspaces
        a.learn_rollout(ro)
        ro.t = T
    torch.cuda.synchronize()
    ms = {k: [] for k in agents}
    peak = {}
    for _ in range(repeats):
        for k, a in agents.items():
            torch.cuda.reset_peak_memory_stats()
            t, _ = _timed(lambda: a.learn_rollout(ro))
            peak[k] = torch.cuda.max_memory_allocated() / 2 ** 20
            ro.t = T
            ms[k].append(t)
    n_mb = s["epochs"] * (s["N"] * T // s["B"])
    out = {"shape": name, **{k: v for k, v in s.items() if k != "net"}, "minibatches_per_learn": n_mb,
           "memory_allocated_mib_all_agents": torch.cuda.memory_allocated() / 2 ** 20}
    for k, a in agents.items():
        out[k] = {"learn_ms_best": min(ms[k]), "learn_ms": ms[k], "us_per_minibatch_best": 1e3 * min(ms[k]) / n_mb,
                  "launches_per_minibatch": a.LAUNCHES_PER_MINIBATCH, "peak_mib_in_learn": peak[k]}
    del agents, ro
    torch.cuda.empty_cache()
    return out


def frames_case(N, rounds=3):
    import time
    import torch
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    T = 128
    env = Env("seaquest", num_envs=N, seed=0, device="cuda")
    agent = Agent("rnd_ppo", state_size=[4, 84, 84], action_size=env.action_size, hidden_size=512, head="cnn",
                  rnd_network="rnd_cnn", obs_normalize=False, n_step=T, batch_size=256, n_epoch=3,
                  optim_config={"name": "adam", "lr": 2.5e-4}, run_step=10 ** 9, lr_decay=False, device="cuda")
    col = RolloutCollector(env, agent)
    agent.learn_rollout(col.collect())                 # warm-up: graph capture, workspaces
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ts = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        agent.learn_rollout(col.collect())
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    res = {"envs": N, "T": T, "A": env.action_size, "seconds": ts, "env_steps_per_s_best": N * T / min(ts),
           "peak_mib": torch.cuda.max_memory_allocated() / 2 ** 20}
    del agent, col, env
    torch.cuda.empty_cache()
    return res


def kernel_times():
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    out = {}
    s = stream_ptr()
    A = 2
    for B in (256, 2048):
        NT = 4 * B
        o = torch.randn(B, A + 2, device="cuda")
        po = o[:, :A + 1].contiguous()
        idx = torch.randperm(NT, device="cuda")[:B].to(torch.int32)
        act = torch.randint(0, A, (NT,), dtype=torch.int32, device="cuda")
        adv, ret, v, ret_i, v_i = (torch.randn(NT, device="cuda") for _ in range(5))
        lpo = -torch.rand(NT, device="cuda")
        dout, pdout = torch.empty(B, A + 2, device="cuda"), torch.empty(B, A + 1, device="cuda")
        stats = torch.empty(8 + 4 * ((B + 255) // 256), device="cuda")
        out[f"rnd_ppo_loss_us_B{B}"] = _events(lambda: C.jb_rnd_ppo_loss(
            0, ptr(o), ptr(idx), ptr(act), ptr(adv), ptr(ret), ptr(v), ptr(ret_i), ptr(v_i), ptr(lpo), B, A, A + 2, 0.1,
            1.0, 0.01, ptr(dout), ptr(stats), 0, s))
        out[f"ppo_loss_us_B{B}"] = _events(lambda: C.jb_ppo_loss(
            0, ptr(po), ptr(idx), ptr(act), ptr(adv), ptr(ret), ptr(v), ptr(lpo), B, A, A + 1, 0.1, 1.0, 0.01, ptr(pdout),
            ptr(stats), 0, s))
        p, t = torch.randn(B, 256, device="cuda"), torch.randn(NT, 256, device="cuda")
        dp = torch.empty(B, 256, device="cuda")
        rstats = torch.empty(1 + (B + 7) // 8, device="cuda")
        out[f"rnd_loss_us_B{B}"] = _events(lambda: C.jb_rnd_loss(ptr(p), ptr(t), ptr(idx), B, 256, 0, ptr(dp), ptr(rstats),
                                                                 0, s))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "rnd_ppo_throughput needs a GPU"
    doc = {"gpu_before": gpu_info()}
    doc["kernels"] = kernel_times()
    doc["learn"] = [learn_case(k, args.repeats) for k in LEARN_SHAPES]
    doc["frames"] = [frames_case(n) for n in (8, 256)]
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
