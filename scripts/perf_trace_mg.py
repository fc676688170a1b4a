"""Intra-step timeline of the persistent PPO kernel WITH the in-kernel gradient exchange (run under torchrun, 2+ ranks):
clock64 stamps of the last step of rank 0 (debug trace, JB_FUSED_SKIP=256)."""
import sys, os, ctypes
os.environ["JB_FUSED_SKIP"] = "256"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.distributed as dist
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
from jorldy_b200.core import Agent, Env, parallel
from jorldy_b200.core.collect import RolloutCollector
from jorldy_b200._lib import C

N, T, B = 4096, 32, 256
env = Env("cartpole", num_envs=N, seed=0, id=rank, device=dev)
agent = Agent("ppo", state_size=4, action_size=2, hidden_size=512, batch_size=B, n_step=T, n_epoch=1,
              optim_config={"name": "adam", "lr": 2.5e-4}, device=dev, run_step=10**9, use_fused=True)
parallel.attach(agent, world)
col = RolloutCollector(env, agent, use_cuda_graph=False); col.collect()
agent.learn_rollout(col.rollout); col.rollout.t = T
st = agent._st; fr = agent._fused[B]
n = N * T // B
for rep in range(3):
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    agent._cursor.zero_(); e0.record(); fr.run(st, n); e1.record(); torch.cuda.synchronize()
    if rank == 0:
        print(f"world {world}: {e0.elapsed_time(e1)/n*1000:.1f} us/step over {n} steps", flush=True)
tr = np.zeros((256, 48), np.int64)
C.jb_ppo_fused_trace(tr.ctypes.data_as(ctypes.c_void_p))
names = {0: "step start", 5: "P1 end", 6: "bar1", 36: "P1 ticket drawn", 37: "row maths done (last arriver)", 38: "row table landed", 40: "critic sums of all ranks", 7: "critic means done",
         16: "JB end", 21: "JA end", 22: "P3 jobs end", 23: "p/m/v issued", 24: "bar3", 41: "X: peers' gradients complete (F1)",
         42: "X: chunk averaged + stored to all ranks", 43: "X: chunk tag published", 44: "X: all chunks of all owners landed",
         25: "P5 fold", 26: "P5 end", 27: "bar5"}
ghz = 1.98                                  # H100 SXM boost clock (clock64 ticks -> us)
if rank == 0:
    for cta in [0, 60, 147]:
        t = tr[cta]
        print(f"--- rank 0 CTA {cta}")
        order = sorted([i for i in names if t[i] > 0], key=lambda i: t[i])
        prev = t[0]
        for i in order:
            print(f"  {names[i]:42s} +{(t[i]-prev)/ghz/1000:6.2f} us   @{(t[i]-t[0])/ghz/1000:6.2f}")
            prev = t[i]
dist.barrier(); torch.cuda.synchronize(); sys.stdout.flush(); os._exit(0)
