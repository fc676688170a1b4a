"""Throughput of the Munchausen agents (M-DQN, M-IQN) on one GPU, in one process, against DQN and IQN:

  learn_*       ms per eager learn() of M-DQN against DQN and of M-IQN against IQN on the same replay (random transitions),
                alternating in blocks of 5 in the same call: CartPole (config.<agent>.cartpole, H=512) and synthetic
                seaquest frames with the CNN head (config.<agent>.atari, 18 actions); B = 32, N = 64
  collect_*     config.<agent>.atari on synthetic seaquest through ReplayCollector with a 1M-slot single-frame replay, 16
                and 256 lanes, the config's update_period env steps per lane and one learn() per round; env-steps/s
  loss_*        jb_mdqn_loss / jb_munchausen_quantile_loss (loss, gradient and stats) against the same maths in torch ops
                (autograd) on the GPU, at the Atari shape (B = 32, A = 18, N = 64), CUDA events over `--iters` calls each,
                alternating in blocks

Also printed: the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after.

  python scripts/munchausen_throughput.py [--learns 50] [--rounds 20] [--iters 200]
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

PAIRS = (("m_dqn", "dqn"), ("m_iqn", "iqn"))


def learn_pair(pair, env_name, learns):
    import numpy as np
    import torch
    from jorldy_b200.core import Env
    atari = env_name != "cartpole"
    env = Env(env_name, num_envs=4, seed=0, device="cuda")
    n = 4096
    agents = []
    for name in pair:
        rs = np.random.RandomState(0)
        _, agent = _agent(f"config.{name}.{'atari' if atari else 'cartpole'}", env, buffer_size=n)
        shape = (n, 4, 84, 84) if atari else (n, 4)
        mk = (lambda: rs.randint(0, 256, size=shape).astype(np.uint8)) if atari else \
            (lambda: rs.standard_normal(shape).astype(np.float32))
        agent.memory.store([{"state": mk(), "next_state": mk(), "action": rs.randint(env.action_size, size=(n, 1)),
                             "reward": rs.standard_normal((n, 1)), "done": rs.uniform(size=(n, 1)) < 0.05}])
        for _ in range(5):
            agent.learn()
        agents.append(agent)
    ts = {name: [] for name in pair}
    for _ in range(max(1, learns // 5)):
        for name, agent in zip(pair, agents):
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                agent.learn()                           # ends in the host read of the stats: synchronised
                ts[name].append((time.perf_counter() - t0) * 1e3)
    out = {"case": f"learn_{pair[0]}_vs_{pair[1]}_{env_name}", "batch_size": agents[0].batch_size,
           "actions": env.action_size}
    for name in pair:
        t = sorted(ts[name])
        out[f"ms_learn_median_{name}"], out[f"ms_learn_best_{name}"] = t[len(t) // 2], t[0]
    return out


def _torch_mdqn(q_all, qt_s, qt_next, action, reward, done, gamma, alpha, tau, l0):
    import torch
    B = q_all.shape[0]
    ar = torch.arange(B, device=q_all.device)
    with torch.no_grad():
        z = qt_s - qt_s.max(1, keepdim=True).values
        tlp = z - tau * torch.logsumexp(z / tau, 1, keepdim=True)
        bonus = alpha * tlp[ar, action].clamp(l0, 0)
        zn = qt_next - qt_next.max(1, keepdim=True).values
        tlpn = zn - tau * torch.logsumexp(zn / tau, 1, keepdim=True)
        v = (torch.softmax(qt_next / tau, 1) * (qt_next - tlpn)).sum(1)
        y = reward + bonus + (1 - done) * gamma * v
    loss = torch.nn.functional.smooth_l1_loss(q_all[ar, action], y)
    loss.backward()
    return loss


def _torch_miqn(theta_all, cur, nxt, action, reward, done, tau_fr, gamma, alpha, tau, l0):
    """theta_all / cur / nxt [B, A, n] views."""
    import torch
    B = theta_all.shape[0]
    ar = torch.arange(B, device=theta_all.device)
    with torch.no_grad():
        qs, qn = cur.mean(2), nxt.mean(2)
        z = qs - qs.max(1, keepdim=True).values
        bonus = alpha * (z - tau * torch.logsumexp(z / tau, 1, keepdim=True))[ar, action].clamp(l0, 0)
        zn = qn - qn.max(1, keepdim=True).values
        tlpn = zn - tau * torch.logsumexp(zn / tau, 1, keepdim=True)
        v = (torch.softmax(qn / tau, 1).unsqueeze(2) * (nxt - tlpn.unsqueeze(2))).sum(1)
        y = (reward + bonus).view(B, 1) + ((1 - done) * gamma).view(B, 1) * v
    theta = theta_all[ar, action]
    u = y.unsqueeze(1) - theta.unsqueeze(2)
    huber = torch.nn.functional.smooth_l1_loss(y.unsqueeze(1).expand_as(u), theta.unsqueeze(2).expand_as(u), reduction="none")
    t = tau_fr.unsqueeze(2)
    loss = torch.where(u < 0, (1 - t) * huber, t * huber).sum(1).mean(1).mean()
    loss.backward()
    return loss


def loss_case(kind, iters):
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B, A, N = 32, 18, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    action = torch.randint(A, (B,), device="cuda", generator=g)
    reward, done = rnd(B), torch.zeros(B, device="cuda")
    stats, scratch = torch.empty(4, device="cuda"), torch.empty(2 * B, device="cuda")
    hp = (0.99, 0.9, 0.03, -1.0)
    if kind == "mdqn":
        q, qs, qn = rnd(B, A), rnd(B, A), rnd(B, A)
        out = torch.empty_like(q)
        leaf = q.clone().requires_grad_(True)

        def cuda():
            C.jb_mdqn_loss(ptr(q), ptr(qs), ptr(qn), ptr(action), 0, ptr(reward), ptr(done), B, A, *hp, ptr(out), ptr(stats),
                           ptr(scratch), stream_ptr())

        def torch_ops():
            leaf.grad = None
            _torch_mdqn(leaf, qs, qn, action, reward, done, *hp)
        view = lambda x: x
    else:
        pred, cur, nxt = rnd(B, N, A), rnd(B, N, A), rnd(B, N, A)
        fr = torch.rand(B, N, device="cuda", generator=g)
        out = torch.empty_like(pred)
        leaf = pred.clone().requires_grad_(True)
        view = lambda x: x.transpose(1, 2)

        def cuda():
            C.jb_munchausen_quantile_loss(ptr(pred), ptr(nxt), ptr(cur), ptr(fr), N, ptr(action), 0, ptr(reward), ptr(done),
                                          B, A, N, N, N, *hp, ptr(out), ptr(stats), ptr(scratch), stream_ptr())

        def torch_ops():
            leaf.grad = None
            _torch_miqn(view(leaf), view(cur), view(nxt), action, reward, done, fr, *hp)

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
    gerr = (view(leaf.grad) - view(out)).abs().max().item()
    return {"case": f"loss_{kind}", "B": B, "A": A, "N": N if kind == "miqn" else None,
            "us_cuda_median": tc[len(tc) // 2], "us_torch_ops_median": tt[len(tt) // 2], "max_abs_grad_diff": gerr}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--learns", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("munchausen_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    for kind in ("mdqn", "miqn"):
        print(json.dumps(loss_case(kind, args.iters)), flush=True)
    for pair in PAIRS:
        for env in ("cartpole", "seaquest"):
            print(json.dumps(learn_pair(pair, env, args.learns)), flush=True)
    for agent in ("m_dqn", "m_iqn"):
        for lanes in (16, 256):
            print(json.dumps(collect_case(agent, lanes, args.rounds, args.warmup)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
