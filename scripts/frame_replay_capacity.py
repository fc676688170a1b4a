"""Capacity and rate of the single-frame Atari replay (jorldy_b200/core/buffer/frame_store.py) at the reference's replay
sizes, on one GPU:

  ape_x_2M_128   config.ape_x.atari (2M slots, 128 actors, batch 512, update_period 100)
  ape_x_2M_256   the same replay behind 256 actors
  rainbow_1M_64  config.rainbow.atari (1M slots) behind 64 actors, update_period 4

Each case collects through ReplayCollector until the replay has wrapped (learning off), then runs `--rounds` rounds with
one learn() each, then times learn() alone.  Prints one JSON line per case and one with the GPU's name, power limit and SM
clock (read-only nvidia-smi query).  The duplicated stack layout needs 56,448 B per slot (112.9 GB at 2M slots).

  python scripts/frame_replay_capacity.py [--cases ape_x_2M_128,...] [--rounds 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = {"ape_x_2M_128": ("config.ape_x.atari", 128, 2_000_000, 100),
         "ape_x_2M_256": ("config.ape_x.atari", 256, 2_000_000, 100),
         "rainbow_1M_64": ("config.rainbow.atari", 64, 1_000_000, 4)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired) as e:
        return {"nvidia_smi": f"unavailable: {e}"}
    return {"nvidia_smi": dict(zip(q.split(","), [x.strip() for x in out[0].split(",")])) if out else None}


def run_case(name, rounds):
    import torch
    from jorldy_b200 import config as cfgs
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.buffer.frame_store import store_bytes
    from jorldy_b200.core.collect import ReplayCollector
    path, lanes, capacity, update_period = CASES[name]
    cfg = cfgs.load(path)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(0)
    env = Env("breakout", num_envs=lanes, seed=0, device="cuda")
    kw = dict(cfg.agent)
    kw.pop("name")
    kw.update(buffer_size=capacity, start_train_step=10 ** 12, num_workers=lanes, run_step=cfg.train["run_step"])
    if cfg.train.get("distributed_batch_size"):
        kw["batch_size"] = cfg.train["distributed_batch_size"]
    agent = Agent(cfg.agent["name"], state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim, **kw)
    rc = ReplayCollector(env, agent, update_period)
    assert rc.frames is not None, "the collector did not attach a frame store"
    mem = agent.memory
    # fill past wrap-around: every slot written at least once and the oldest overwritten
    step, t0 = 0, time.perf_counter()
    while mem.buffer_counter < capacity or step * lanes < capacity + lanes * update_period:
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    fill_sec = time.perf_counter() - t0
    fill_rate = step * lanes / fill_sec
    agent.start_train_step = 0
    step, _ = rc.run_round(step)                 # warm-up learn
    torch.cuda.synchronize()
    s0, t0 = step, time.perf_counter()
    results = []
    for _ in range(rounds):
        step, r = rc.run_round(step)
        results.append(bool(r))
    torch.cuda.synchronize()
    train_rate = (step - s0) * lanes / (time.perf_counter() - t0)
    times = []
    for _ in range(10):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        agent.learn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    mem.check_frames()
    out = {"case": name, "config": path, "lanes": lanes, "replay_slots": capacity, "update_period": update_period,
           "batch_size": agent.batch_size, "frames_per_lane": rc.frames.F,
           "frame_store_bytes": store_bytes(capacity, lanes, agent.n_step), "replay_slots_written": step * lanes,
           "wrapped": step * lanes > capacity, "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(),
           "fill_env_steps_per_sec": fill_rate, "train_env_steps_per_sec": train_rate, "rounds_with_learn": sum(results),
           "rounds_timed": rounds, "ms_per_learn": sorted(times)[len(times) // 2], "status_word": int(rc.frames.status[0])}
    del rc, agent, env, mem
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("frame_replay_capacity.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    for name in args.cases.split(","):
        print(json.dumps(run_case(name, args.rounds)), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
