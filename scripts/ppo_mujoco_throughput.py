"""Throughput of PPO on the synthetic MuJoCo tasks at config.ppo.mujoco's sizes (32 envs, T=2048, B=512, 10 epochs,
H=512), on one GPU, in one process.  hopper (obs 11) runs the persistent minibatch kernel (csrc/ppo_fused.cu, inputs
<= 16); walker and half_cheetah (obs 17) run the CUDA-graph multi-launch path, so the difference is what the 17-dim
tasks pay until the persistent kernel takes wider inputs.

Each task runs one collect() + learn_rollout() as warm-up, then the tasks alternate for --repeats rounds of one timed
collect() and one timed learn_rollout() (CUDA events); reported per task: the best and the spread of env steps per
second (collect + learn) and of ms per minibatch step (learn / (epochs x minibatches)), and which learner path ran.
Also printed: the GPU's name, power limit and SM clock (read-only nvidia-smi query).

  python scripts/ppo_mujoco_throughput.py [--repeats 3] [--tasks hopper,walker,half_cheetah]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from frame_replay_capacity import gpu_info  # noqa: E402
from ppo_frames_throughput import _timed  # noqa: E402

N, T, B, EPOCHS, H = 32, 2048, 512, 10, 512


def _setup(task):
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    env = Env(task, num_envs=N, seed=0, device="cuda")
    agent = Agent("ppo", state_size=env.state_size, action_size=env.action_size, hidden_size=H,
                  network="continuous_policy_value", n_step=T, batch_size=B, n_epoch=EPOCHS,
                  optim_config={"name": "adam", "lr": 3e-4}, run_step=10 ** 9, lr_decay=False, device="cuda")
    col = RolloutCollector(env, agent)
    agent.learn_rollout(col.collect())                  # warm-up: graph capture of collect and of the minibatch chunk
    return agent, col


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--tasks", type=str, default="hopper,walker,half_cheetah")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ppo_mujoco_throughput.py measures on a CUDA device; none is available")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), **gpu_info()}), flush=True)
    tasks = args.tasks.split(",")
    runs = {t: _setup(t) for t in tasks}
    torch.cuda.synchronize()
    times = {t: ([], []) for t in tasks}
    for _ in range(args.repeats):
        for t in tasks:
            agent, col = runs[t]
            c_ms, ro = _timed(col.collect)
            l_ms, _ = _timed(lambda: agent.learn_rollout(ro))
            times[t][0].append(c_ms)
            times[t][1].append(l_ms)
    n_mb = EPOCHS * (N * T // B)
    for t in tasks:
        agent, _ = runs[t]
        tot = [c + l for c, l in zip(*times[t])]
        tl = times[t][1]
        sps = [N * T / (x / 1e3) for x in tot]
        print(json.dumps({"task": t, "obs": agent.state_size, "act": agent.action_size, "envs": N, "T": T,
                          "batch_size": B, "n_epoch": EPOCHS, "hidden": H,
                          "learner": "persistent" if agent._fused else "graph multi-launch",
                          "env_steps_per_sec_best": max(sps), "env_steps_per_sec_spread": max(sps) - min(sps),
                          "ms_per_minibatch_best": min(tl) / n_mb, "ms_per_minibatch_spread": (max(tl) - min(tl)) / n_mb,
                          "ms_collect": times[t][0], "ms_learn": tl}), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
