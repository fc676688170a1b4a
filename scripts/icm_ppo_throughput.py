"""ICM-PPO against PPO's multi-launch path on one GPU, in one process; prints one JSON document.

  learn   learn_rollout() ms of ICM-PPO and of PPO with use_fused=False (the CUDA-graph multi-launch path ICM-PPO
          shares) on the same collected rollout, alternated for --repeats rounds, at the ppo_cartpole benchmark shape
          (4096 CartPole envs, T = 128, B = 256, 3 epochs, H = 512) and at Hopper dimensions with config.ppo.mujoco's
          sizes (32 envs, T = 2048, B = 512, 10 epochs, H = 512); launches per minibatch and peak memory of each
  kernels jb_icm_loss (with its finalize) at B = 256 / 2048 and the reward-only pass over 524 288 rows, and
          jb_bn_elu_fwd / jb_bn_elu_bwd at M = 256, 2048 and 524 288 (N = 256), CUDA events over 100 launches
  frames  collect + learn env steps/s of ICM-PPO on synthetic Atari frames (CNN head and CNN ICM, A = 18, T = 128,
          B = 256, 3 epochs, H = 512) at 8 and 256 envs, and peak memory
  gpu     name, power limit and SM clock (read-only nvidia-smi query), read before and after

  python scripts/icm_ppo_throughput.py [--repeats 3] [--out PATH]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402
from ppo_frames_throughput import _timed  # noqa: E402

LEARN_SHAPES = {
    "ppo_cartpole": dict(env="cartpole", N=4096, T=128, B=256, epochs=3, lr=2.5e-4, net="discrete_policy_value"),
    "hopper": dict(env="hopper", N=32, T=2048, B=512, epochs=10, lr=3e-4, net="continuous_policy_value"),
}


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
    agents = {"icm_ppo": mk("icm_ppo"), "ppo_multilaunch": mk("ppo", use_fused=False)}
    agents["ppo_multilaunch"].network.load_state_dict(agents["icm_ppo"].network.state_dict())
    ro = RolloutCollector(env, agents["icm_ppo"]).collect()      # keeps next_state; PPO reads only what it always did
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
    out = {"shape": name, **{k: v for k, v in s.items() if k != "net"}, "minibatches_per_learn": n_mb}
    for k, a in agents.items():
        out[k] = {"learn_ms_best": min(ms[k]), "learn_ms": ms[k], "us_per_minibatch_best": 1e3 * min(ms[k]) / n_mb,
                  "launches_per_minibatch": a.LAUNCHES_PER_MINIBATCH, "peak_mib_in_learn": peak[k]}
    return out


def frames_case(N, rounds=3):
    import time
    import torch
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    T = 128
    env = Env("seaquest", num_envs=N, seed=0, device="cuda")
    agent = Agent("icm_ppo", state_size=[4, 84, 84], action_size=env.action_size, hidden_size=512, head="cnn",
                  icm_network="icm_cnn", obs_normalize=False, n_step=T, batch_size=256, n_epoch=3,
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
    return {"envs": N, "T": T, "A": env.action_size, "seconds": ts, "env_steps_per_s_best": N * T / min(ts),
            "peak_mib": torch.cuda.max_memory_allocated() / 2 ** 20}


def _events(fn, n=100):
    import torch
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return 1e3 * a.elapsed_time(b) / n


def kernel_times():
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    out = {}
    s = stream_ptr()
    for B in (256, 2048, 524288):
        f = torch.randn(B, 256, device="cuda")
        pp = torch.randn(B, 512, device="cuda")
        g = torch.randn(B, 2, device="cuda")
        act = torch.randint(0, 2, (B,), dtype=torch.int32, device="cuda")
        ri, df, dg = torch.empty(B, device="cuda"), torch.empty(B, 256, device="cuda"), torch.empty(B, 2, device="cuda")
        stats = torch.empty(4 + 3 * ((B + 7) // 8), device="cuda")
        if B == 524288:
            out["icm_loss_reward_only_us_M524288"] = _events(lambda: C.jb_icm_loss(
                0, ptr(f), ptr(pp[:, 256:]), 512, 0, 0, 0, B, 2, 256, 0.01, 0.2, ptr(ri), 0, 0, 0, 0, s))
        else:
            out[f"icm_loss_us_B{B}"] = _events(lambda: C.jb_icm_loss(
                0, ptr(f), ptr(pp[:, 256:]), 512, ptr(g), 0, ptr(act), B, 2, 256, 0.01, 0.2, 0, ptr(df), ptr(dg),
                ptr(stats), 0, s))
    N = 256
    for M in (256, 2048, 524288):
        x, dy = torch.randn(M, N, device="cuda"), torch.randn(M, N, device="cuda")
        y, dx, xhat = (torch.empty(M, N, device="cuda") for _ in range(3))
        gam, bet = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
        rm, rv = torch.zeros(N, device="cuda"), torch.ones(N, device="cuda")
        nbt = torch.zeros((), dtype=torch.int64, device="cuda")
        mean, inv, dgam, dbet = (torch.empty(N, device="cuda") for _ in range(4))
        part = torch.empty(C.jb_col_partials_doubles(M, N), dtype=torch.float64, device="cuda")
        out[f"bn_elu_fwd_us_M{M}"] = _events(lambda: C.jb_bn_elu_fwd(
            ptr(x), M, N, ptr(gam), ptr(bet), ptr(rm), ptr(rv), ptr(nbt), 0.1, 1e-5, ptr(mean), ptr(inv), ptr(part),
            ptr(y), N, 0, 0, s))
        out[f"bn_elu_bwd_us_M{M}"] = _events(lambda: C.jb_bn_elu_bwd(
            ptr(dy), N, ptr(y), N, ptr(x), M, N, ptr(gam), ptr(mean), ptr(inv), ptr(xhat), ptr(part), ptr(dx), ptr(dgam),
            ptr(dbet), s))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "icm_ppo_throughput needs a GPU"
    doc = {"gpu_before": gpu_info()}
    doc["learn"] = [learn_case(k, args.repeats) for k in LEARN_SHAPES]
    doc["kernels"] = kernel_times()
    doc["frames"] = [frames_case(n) for n in (8, 256)]
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
