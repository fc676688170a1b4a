"""Throughput of the Rainbow-IQN agent on one GPU, in one process, against Rainbow and IQN:

  learn_*       ms per eager learn() of rainbow_iqn, rainbow and iqn on the same kind of replay (random transitions, n-step
                windows for the n-step agents), alternating in blocks of 5 in the same call: CartPole (config.<agent>.cartpole,
                H=512) and synthetic seaquest frames with the CNN head (config.<agent>.atari, 18 actions); B = 32, N = 64
  loss          jb_rainbow_iqn_loss (a*, n-step targets, weighted loss, gradient, priorities, stats) against the same maths in
                torch ops (autograd) on the GPU, at the Atari shape (B = 32, A = 18, N = 64, n = 3), CUDA events over
                `--iters` calls each, alternating in blocks
  collect_*     config.rainbow_iqn.atari on synthetic seaquest through ReplayCollector with a 1M-slot single-frame replay, 16
                and 256 lanes, the config's update_period env steps per lane and at most one learn() per round; env-steps/s

Also printed: the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after.

  python scripts/rainbow_iqn_throughput.py [--learns 50] [--rounds 20] [--iters 200]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402
from quantile_throughput import _agent, collect_case  # noqa: E402

AGENTS = ("rainbow_iqn", "rainbow", "iqn")


def learn_block(env_name, learns):
    import numpy as np
    import torch
    from jorldy_b200.core import Env
    atari = env_name != "cartpole"
    env = Env(env_name, num_envs=4, seed=0, device="cuda")
    n = 4096
    agents = []
    for name in AGENTS:
        rs = np.random.RandomState(0)
        _, agent = _agent(f"config.{name}.{'atari' if atari else 'cartpole'}", env, buffer_size=n)
        k = agent.n_step
        shape = (n, 4, 84, 84) if atari else (n, 4)
        mk = (lambda: rs.randint(0, 256, size=shape).astype(np.uint8)) if atari else \
            (lambda: rs.standard_normal(shape).astype(np.float32))
        agent.memory.store([{"state": mk(), "next_state": mk(), "action": rs.randint(env.action_size, size=(n, 1)),
                             "reward": rs.standard_normal((n, k, 1) if k > 1 else (n, 1)),
                             "done": rs.uniform(size=(n, k, 1) if k > 1 else (n, 1)) < 0.05}])
        for _ in range(5):
            agent.learn()
        agents.append(agent)
    ts = {name: [] for name in AGENTS}
    for _ in range(max(1, learns // 5)):
        for name, agent in zip(AGENTS, agents):
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                agent.learn()                           # ends in the host read of the stats: synchronised
                ts[name].append((time.perf_counter() - t0) * 1e3)
    out = {"case": f"learn_{env_name}", "batch_size": agents[0].batch_size, "actions": env.action_size,
           "quantiles": agents[0].num_sample}
    for name in AGENTS:
        t = sorted(ts[name])
        out[f"ms_learn_median_{name}"], out[f"ms_learn_best_{name}"] = t[len(t) // 2], t[0]
    return out


def _torch_loss(theta_all, next_online, next_target, action, reward, done, weights, tau_fr, gamma, alpha):
    """[B, N, A] tensors; reward / done [B, n]; returns (loss, priorities) and fills theta_all.grad."""
    import torch
    B = theta_all.shape[0]
    ar = torch.arange(B, device=theta_all.device)
    with torch.no_grad():
        a_star = next_online.mean(1).argmax(1)
        y = next_target[ar, :, a_star]
        for s in reversed(range(reward.shape[1])):
            y = reward[:, s:s + 1] + (1 - done[:, s:s + 1]) * gamma * y
    theta = theta_all[ar, :, action]
    u = y.unsqueeze(1) - theta.unsqueeze(2)
    huber = torch.nn.functional.smooth_l1_loss(y.unsqueeze(1).expand_as(u), theta.unsqueeze(2).expand_as(u), reduction="none")
    t = tau_fr.unsqueeze(2)
    per = torch.where(u < 0, (1 - t) * huber, t * huber).sum(1).mean(1)
    loss = (weights.to(per.dtype) * per).mean()
    loss.backward()
    return loss, per.detach().to(torch.float64) ** alpha


def loss_case(iters):
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B, A, N, n = 32, 18, 64, 3
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    action = torch.randint(A, (B,), device="cuda", generator=g)
    reward, done = rnd(B, n), (torch.rand(B, n, device="cuda", generator=g) < 0.1).float()
    weights = torch.rand(B, device="cuda", generator=g, dtype=torch.float64) * 0.9 + 0.1
    pred, nxt_on, nxt_tg = rnd(B, N, A), rnd(B, N, A), rnd(B, N, A)
    fr = torch.rand(B, N, device="cuda", generator=g)
    out, loss = torch.empty_like(pred), torch.empty(B, device="cuda")
    prio, stats, scratch = torch.empty(B, device="cuda", dtype=torch.float64), torch.empty(4, device="cuda"), \
        torch.empty(4 * B, device="cuda")
    leaf = pred.clone().requires_grad_(True)

    def cuda():
        C.jb_rainbow_iqn_loss(ptr(pred), ptr(nxt_on), ptr(nxt_tg), ptr(fr), ptr(action), 0, ptr(reward), ptr(done),
                              ptr(weights), B, A, N, N, N, n, 0.99, 0.5, ptr(out), ptr(loss), ptr(prio), None, ptr(stats),
                              ptr(scratch), stream_ptr())

    def torch_ops():
        leaf.grad = None
        return _torch_loss(leaf, nxt_on, nxt_tg, action, reward, done, weights, fr, 0.99, 0.5)

    def timed(fn, k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / k * 1e3

    for fn in (cuda, torch_ops):
        timed(fn, 20)
    tc, tt = [], []
    for _ in range(10):
        tc.append(timed(cuda, iters // 10))
        tt.append(timed(torch_ops, iters // 10))
    tc.sort(), tt.sort()
    cuda()
    _, p_ref = torch_ops()
    torch.cuda.synchronize()
    return {"case": "loss_rainbow_iqn", "B": B, "A": A, "N": N, "n_step": n, "us_cuda_median": tc[len(tc) // 2],
            "us_torch_ops_median": tt[len(tt) // 2], "max_abs_grad_diff": (leaf.grad - out).abs().max().item(),
            "max_rel_prio_diff": ((prio - p_ref).abs() / p_ref).max().item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("rainbow_iqn_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    print(json.dumps(loss_case(args.iters)), flush=True)
    for env in ("cartpole", "seaquest"):
        print(json.dumps(learn_block(env, args.learns)), flush=True)
    for lanes in (16, 256):
        print(json.dumps(collect_case("rainbow_iqn", lanes, args.rounds, args.warmup)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
