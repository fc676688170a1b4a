"""V-MPO against PPO on one GPU, in one process; prints one JSON document.

  learn   learn_rollout() ms of V-MPO and of PPO (its default path, and use_fused=False: the CUDA-graph multi-launch
          path V-MPO shares) on the same collected rollout, the three agents alternated for --repeats rounds, at the
          ppo_cartpole benchmark shape (4096 CartPole envs, T = 128, B = 256, 3 epochs, H = 512) and at Hopper
          dimensions with config.ppo.mujoco's sizes (32 envs, T = 2048, B = 512, 10 epochs, H = 512)
  loss    jb_vmpo_loss against jb_ppo_loss (each with its finalize launch), CUDA events over 200 launches, at B = 256
          and B = 2048 (discrete A = 2 and continuous A = 3)
  frames  collect + learn env steps/s of V-MPO on synthetic Atari frames (CNN head, A = 18) at 8 and 1024 envs
  gpu     name, power limit and SM clock (read-only nvidia-smi query), read before and after

  python scripts/vmpo_throughput.py [--repeats 3]
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
    agents = {"vmpo": mk("vmpo"), "ppo": mk("ppo"), "ppo_multilaunch": mk("ppo", use_fused=False)}
    for a in agents.values():
        a.network.load_state_dict(agents["vmpo"].network.state_dict())
    col = RolloutCollector(env, agents["ppo"])
    ro = col.collect()
    T = s["T"]
    for a in agents.values():                         # warm-up: graph capture, workspaces
        a.learn_rollout(ro)
        ro.t = T
    torch.cuda.synchronize()
    ms = {k: [] for k in agents}
    for _ in range(repeats):
        for k, a in agents.items():
            t, _ = _timed(lambda: a.learn_rollout(ro))
            ro.t = T
            ms[k].append(t)
    n_mb = s["epochs"] * (s["N"] * T // s["B"])
    out = {"shape": name, **{k: v for k, v in s.items() if k != "net"}, "minibatches_per_learn": n_mb}
    for k, a in agents.items():
        out[k] = {"learn_ms_best": min(ms[k]), "learn_ms": ms[k], "us_per_minibatch_best": 1e3 * min(ms[k]) / n_mb,
                  "path": "persistent" if a._fused else "graph multi-launch"}
    return out


def loss_case(B, cont, iters=200):
    import numpy as np
    import torch
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    A = 3 if cont else 2
    nout = 2 * A + 1 if cont else A + 1
    NT = 4 * B
    rs = np.random.RandomState(B)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out, out_old = t(rs.standard_normal((B, nout)).astype(np.float32)), t(rs.standard_normal((NT, nout)).astype(np.float32))
    idx = t(rs.permutation(NT)[:B].astype(np.int32))
    action = t(rs.uniform(-0.9, 0.9, (NT, A)).astype(np.float32)) if cont else t(rs.randint(0, A, NT).astype(np.int32))
    adv, ret, vold = (t(rs.standard_normal(NT).astype(np.float32)) for _ in range(3))
    lpo = t(rs.standard_normal((NT, A if cont else 1)).astype(np.float32) - 1.0)
    mult = t(np.array([1.0, 5.0, 1.0], np.float32))
    dout, dmult = torch.empty(B, nout, device="cuda"), torch.empty(3, device="cuda")
    stats = torch.empty(16 + 4 * ((B + 255) // 256), device="cuda")
    acc = torch.zeros(8, device="cuda")
    s = stream_ptr()
    vmpo = lambda: C.jb_vmpo_loss(int(cont), ptr(out), ptr(out_old), ptr(idx), ptr(action), ptr(adv), ptr(ret), B, A, nout,
                                  ptr(mult), 0.01, 0.01, 5e-5, ptr(dout), ptr(dmult), ptr(stats), ptr(acc), s)
    ppo = lambda: C.jb_ppo_loss(int(cont), ptr(out), ptr(idx), ptr(action), ptr(adv), ptr(ret), ptr(vold), ptr(lpo), B, A,
                                nout, 0.1, 1.0, 0.01, ptr(dout), ptr(stats), ptr(acc), s)
    res = {"B": B, "continuous": cont, "A": A}
    for name, fn in (("vmpo", vmpo), ("ppo", ppo)):
        fn()
        torch.cuda.synchronize()
        samples = []
        for _ in range(5):
            ms, _ = _timed(lambda: [fn() for _ in range(iters)])
            samples.append(1e3 * ms / iters)
        res[f"{name}_us_per_call_best"] = min(samples)
        res[f"{name}_us_per_call"] = samples
    return res


def frames_case(N, repeats):
    import torch
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    env = Env("seaquest", num_envs=N, seed=0, device="cuda")
    T, B = 128, min(256, N * 128 // 4)
    agent = Agent("vmpo", state_size=[4, 84, 84], action_size=env.action_size, hidden_size=512, head="cnn",
                  network="discrete_policy_value", n_step=T, batch_size=B, n_epoch=3, run_step=10 ** 9, lr_decay=False,
                  optim_config={"name": "adam", "lr": 2.5e-4}, device="cuda")
    col = RolloutCollector(env, agent)
    agent.learn_rollout(col.collect())
    torch.cuda.synchronize()
    tot = []
    for _ in range(repeats):
        c_ms, ro = _timed(col.collect)
        l_ms, _ = _timed(lambda: agent.learn_rollout(ro))
        tot.append((c_ms, l_ms))
    sps = [N * T / ((c + l) / 1e3) for c, l in tot]
    return {"envs": N, "T": T, "batch_size": B, "n_epoch": 3, "action_size": env.action_size,
            "env_steps_per_sec_best": max(sps), "env_steps_per_sec": sps, "ms_collect_learn": tot}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("vmpo_throughput.py measures on a CUDA device; none is available")
    doc = {"gpu": torch.cuda.get_device_name(0), "gpu_before": gpu_info()}
    doc["loss_kernel"] = [loss_case(B, cont) for B in (256, 2048) for cont in (False, True)]
    doc["learn"] = [learn_case(k, args.repeats) for k in LEARN_SHAPES]
    doc["frames"] = [frames_case(N, args.repeats) for N in (8, 1024)]
    doc["gpu_after"] = gpu_info()
    print(json.dumps(doc), flush=True)


if __name__ == "__main__":
    main()
