"""R2D2 throughput on one GPU, in one process (numbers for DESIGN.md §8).

Reports, with the card's name and power limit read in the same run:
  - ms per eager learn() on CartPole (config.r2d2.cartpole's agent) and on synthetic seaquest at config.r2d2.atari's
    B = 64, L = 40 + 80 + 5, n = 5, CNN head, LSTM 512 (replay filled with random stacked sequences);
  - CUDA-event medians of jb_lstm_step_fwd / jb_lstm_step_bwd (M = 64, H = 512) and jb_r2d2_loss (B 64, T 80, n 5, A 18);
  - collection env-steps/s of config.r2d2.atari (act + env step + frame push + sequence assembly, no learn) at 16 and 256
    lanes;
  - CUDA kernel launches per learn() (torch.profiler, separate run), and peak torch.cuda.max_memory_allocated.
Prints one JSON document; --out PATH also writes it to PATH.
Usage: python scripts/r2d2_throughput.py [--out PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from jorldy_b200 import config as cfg  # noqa: E402
from jorldy_b200._lib import C  # noqa: E402
from jorldy_b200.core import Agent, Env  # noqa: E402
from jorldy_b200.core.collect import ReplayCollector  # noqa: E402

DEV = "cuda"


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def events(fn, iters=50, warm=5):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.percentile(ts, 90))


def agent_for(path, **over):
    c = cfg.load(path)
    a = dict(c.agent)
    a.pop("name")
    a.update(over)
    if path.endswith("atari"):
        D, A = [4, 84, 84], 18
    else:
        D, A = 4, 2
    return Agent("r2d2", state_size=D, action_size=A, optim_config=c.optim, run_step=10 ** 6, device=DEV, seed=0, **a), D, A


def fill(agent, D, A, n, rs):
    L, H = agent.L, agent.network.D_hidden
    for s in range(0, n, 16):
        m = min(16, n - s)
        st = (torch.randint(0, 256, (m, L, 4, 84, 84), dtype=torch.uint8, device=DEV) if isinstance(D, list)
              else torch.randn(m, L, D, device=DEV))
        agent.memory.store([{"state": st, "action": torch.randint(0, A, (m, L), device=DEV),
                             "prev_action": torch.randint(-1, A, (m, L), device=DEV),
                             "reset": (torch.rand(m, L, device=DEV) < 0.01).float(), "reward": torch.randn(m, L, device=DEV),
                             "done": (torch.rand(m, L, device=DEV) < 0.01).float(),
                             "h0": torch.randn(m, H, device=DEV) * 0.1, "c0": torch.randn(m, H, device=DEV) * 0.1}])


def learn_ms(path, cap, **over):
    agent, D, A = agent_for(path, buffer_size=cap, lr_decay=False, **over)
    fill(agent, D, A, cap, np.random.RandomState(0))
    torch.cuda.synchronize()
    for _ in range(3):
        agent.learn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(20):
        t0 = time.perf_counter()
        agent.learn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        agent.learn()
        torch.cuda.synchronize()
    launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                   and "Memset" not in e.name)
    return {"B": agent.batch_size, "L": agent.L, "n": agent.n_step, "H": agent.network.D_hidden,
            "ms_median": float(np.median(ts)), "ms_p90": float(np.percentile(ts, 90)), "cuda_kernels_per_learn": launches}


def kernels():
    B, T, n, A, H = 64, 80, 5, 18, 512
    M, G = B, 4 * H
    r = lambda *s: torch.randn(*s, device=DEV)
    xg, hp, c, w = r(M, G), r(M, H), r(M, H), r(G, H) * 0.04
    h, gates, hpe, dg, dc = r(M, H), r(M, G), r(M, H), r(M, G), r(M, H)
    reset = (torch.rand(M, device=DEV) < 0.1).float()
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    fwd = events(lambda: C.jb_lstm_step_fwd(p(xg), p(hp), p(c), p(w), p(reset), M, H, p(h), p(c), p(gates), p(hpe), s), 200)
    dgn = r(M, G)
    bwd = events(lambda: C.jb_lstm_step_bwd(p(h), p(dgn), p(w), p(gates), p(hp), p(c), p(dc), p(reset), p(reset), M, H, p(dg),
                                            p(dc), s), 200)
    q, qn, qt = r(B, T, A), r(B, T, A), r(B, T, A)
    act = torch.randint(0, A, (B, T), device=DEV)
    rew, done = r(B, T + n), (torch.rand(B, T + n, device=DEV) < 0.05).float()
    wts = torch.rand(B, dtype=torch.float64, device=DEV)
    dq, prio = r(B, T, A), torch.empty(B, dtype=torch.float64, device=DEV)
    st, sc = torch.empty(2, device=DEV), torch.empty(2 * B, dtype=torch.float64, device=DEV)
    loss = events(lambda: C.jb_r2d2_loss(p(q), p(qn), p(qt), p(act), p(rew), p(done), p(wts), B, T, A, n, 0.997, 0.9, 0.9,
                                         p(dq), p(prio), p(st), p(sc), s), 200)
    return {"lstm_step_fwd_us": [1e3 * v for v in fwd], "lstm_step_bwd_us": [1e3 * v for v in bwd],
            "r2d2_loss_us": [1e3 * v for v in loss], "shape": dict(M=M, H=H, B=B, T=T, n=n, A=A)}


def collect_rate(lanes, rounds=6):
    agent, _, _ = agent_for("config.r2d2.atari", buffer_size=4096, start_train_step=10 ** 12)
    env = Env("seaquest", num_envs=lanes, seed=0, device=DEV)
    rc = ReplayCollector(env, agent, update_period=100)
    step = 0
    step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    return lanes * 100 * rounds / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON document to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("r2d2_throughput.py measures the GPU; no CUDA device found")
    out = {"card": card()}
    torch.cuda.reset_peak_memory_stats()
    out["learn_cartpole"] = learn_ms("config.r2d2.cartpole", 1024)
    out["learn_atari"] = learn_ms("config.r2d2.atari", 192)
    out["kernels"] = kernels()
    out["collect_env_steps_per_s"] = {str(n): collect_rate(n) for n in (16, 256)}
    out["peak_max_memory_allocated_GB"] = torch.cuda.max_memory_allocated() / 2 ** 30
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
