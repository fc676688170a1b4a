"""Throughput of the quantile agents (QR-DQN, IQN) on one GPU, in one process:

  learn_*       ms per eager learn() on a replay filled with random transitions: CartPole (config.<agent>.cartpole, H=512)
                and synthetic seaquest frames with the CNN head (config.<agent>.atari, 18 actions); B = 32, K = 200 / N = 64
  collect_*     config.<agent>.atari on synthetic seaquest through ReplayCollector with a 1M-slot single-frame replay, 16
                and 256 lanes, the config's update_period env steps per lane and one learn() per round; env-steps/s
                counts every lane's steps over the timed rounds
  loss_*        jb_quantile_loss (loss, gradient and stats) against the same loss and gradient written in torch ops
                (autograd) on the GPU, at the Atari shape, CUDA events over `--iters` calls each, alternating in blocks

Also printed: the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after.

  python scripts/quantile_throughput.py [--learns 50] [--rounds 20] [--iters 200]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402


def _agent(path, env, **over):
    from jorldy_b200 import config as cfgs
    from jorldy_b200.core import Agent
    cfg = cfgs.load(path)
    ag = dict(cfg.agent, start_train_step=0, lr_decay=False, **over)
    return cfg, Agent(**dict(ag, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
                             run_step=10 ** 9, device="cuda"))


def learn_case(agent_name, env_name, learns):
    import numpy as np
    import torch
    from jorldy_b200.core import Env
    atari = env_name != "cartpole"
    env = Env(env_name, num_envs=4, seed=0, device="cuda")
    rs, n = np.random.RandomState(0), 4096
    cfg, agent = _agent(f"config.{agent_name}.{'atari' if atari else 'cartpole'}", env, buffer_size=n)
    shape = (n, 4, 84, 84) if atari else (n, 4)
    mk = (lambda: rs.randint(0, 256, size=shape).astype(np.uint8)) if atari else (lambda: rs.standard_normal(shape).astype(np.float32))
    agent.memory.store([{"state": mk(), "next_state": mk(), "action": rs.randint(env.action_size, size=(n, 1)),
                         "reward": rs.standard_normal((n, 1)), "done": rs.uniform(size=(n, 1)) < 0.05}])
    for _ in range(5):
        agent.learn()
    ts = []
    for _ in range(learns):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        agent.learn()                                   # ends in the host read of the stats: synchronised
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return {"case": f"learn_{agent_name}_{env_name}", "batch_size": agent.batch_size, "actions": env.action_size,
            "quantiles": getattr(agent, "num_support", None) or agent.num_sample, "hidden": cfg.agent.get("hidden_size", 512),
            "ms_learn_median": ts[len(ts) // 2], "ms_learn_best": ts[0]}


def collect_case(agent_name, lanes, rounds, warmup):
    import torch
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    from jorldy_b200 import config as cfgs
    cfg = cfgs.load(f"config.{agent_name}.atari")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    env = Env("seaquest", num_envs=lanes, seed=0, device="cuda", **{k: v for k, v in cfg.env.items() if k != "name"})
    _, agent = _agent(f"config.{agent_name}.atari", env)
    period = int(cfg.train["update_period"])
    rc = ReplayCollector(env, agent, period)
    step = 0
    for _ in range(warmup):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        step, res = rc.run_round(step)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"case": f"collect_{agent_name}_{lanes}", "lanes": lanes, "update_period": period,
            "replay_slots": agent.memory.buffer_size, "frame_store": agent.memory.frames is not None,
            "env_steps_per_sec": lanes * period * rounds / dt, "ms_per_round": dt / rounds * 1e3,
            "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(), "last_result": res}


def _torch_loss(theta_all, theta_next, action, reward, done, tau, gamma):
    """The loss and gradient as torch ops: theta_all / theta_next [B, A, N] views, tau [B, N] or [N]."""
    import torch
    B = theta_all.shape[0]
    ar = torch.arange(B, device=theta_all.device)
    with torch.no_grad():
        a_star = theta_next.mean(2).argmax(1)
        y = reward.view(B, 1) + (1 - done.view(B, 1)) * gamma * theta_next[ar, a_star]
    theta = theta_all[ar, action]
    u = y.unsqueeze(1) - theta.unsqueeze(2)
    huber = torch.nn.functional.smooth_l1_loss(y.unsqueeze(1).expand_as(u), theta.unsqueeze(2).expand_as(u), reduction="none")
    t = tau.expand_as(theta).unsqueeze(2)
    loss = torch.where(u < 0, (1 - t) * huber, t * huber).sum(1).mean(1).mean()
    loss.backward()
    return loss


def loss_case(layout, iters):
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B, A, N = 32, 18, (200 if layout == "qrdqn" else 64)
    g = torch.Generator(device="cuda").manual_seed(0)
    shape = (B, A, N) if layout == "qrdqn" else (B, N, A)
    pred = torch.randn(shape, device="cuda", generator=g)
    nxt = torch.randn(shape, device="cuda", generator=g)
    sa, sq = (N, 1) if layout == "qrdqn" else (1, A)
    if layout == "qrdqn":
        tau, stride = (2 * torch.arange(N, device="cuda", dtype=torch.float32) + 1) / (2 * N), 0
    else:
        tau, stride = torch.rand(B, N, device="cuda", generator=g), N
    action = torch.randint(A, (B,), device="cuda", generator=g)
    reward, done = torch.randn(B, device="cuda", generator=g), torch.zeros(B, device="cuda")
    dpred, loss, scratch = torch.empty_like(pred), torch.empty(B, device="cuda"), torch.empty(2 * B, device="cuda")
    stats = torch.empty(4, device="cuda")
    view = (lambda x: x) if layout == "qrdqn" else (lambda x: x.transpose(1, 2))

    def cuda():
        C.jb_quantile_loss(ptr(pred), sa, sq, ptr(nxt), sa, sq, ptr(tau), stride, ptr(action), 0, ptr(reward), ptr(done), B,
                           A, N, N, 0.99, ptr(dpred), ptr(loss), None, ptr(stats), ptr(scratch), stream_ptr())

    leaf = pred.clone().requires_grad_(True)

    def torch_ops():
        leaf.grad = None
        _torch_loss(view(leaf), view(nxt), action, reward, done, tau, 0.99)

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n * 1e3

    for fn in (cuda, torch_ops):
        timed(fn, 20)
    tc, tt = [], []
    for _ in range(10):
        tc.append(timed(cuda, iters // 10))
        tt.append(timed(torch_ops, iters // 10))
    tc.sort(), tt.sort()
    torch_ops()
    gerr = (view(leaf.grad) - view(dpred)).abs().max().item()
    return {"case": f"loss_{layout}", "B": B, "A": A, "N": N, "us_jb_quantile_loss_median": tc[len(tc) // 2],
            "us_torch_ops_median": tt[len(tt) // 2], "max_abs_grad_diff": gerr}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("quantile_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    for layout in ("qrdqn", "iqn"):
        print(json.dumps(loss_case(layout, args.iters)), flush=True)
    for agent in ("qrdqn", "iqn"):
        for env in ("cartpole", "seaquest"):
            print(json.dumps(learn_case(agent, env, args.learns)), flush=True)
    for agent in ("qrdqn", "iqn"):
        for lanes in (16, 256):
            print(json.dumps(collect_case(agent, lanes, args.rounds, args.warmup)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
