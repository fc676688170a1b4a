"""Multi-GPU learner plumbing: one process per GPU, torch.distributed (NCCL over NVLink 5 /
NVSwitch) for the only real exchange step of the PPO path — the gradient all-reduce between
backward and the clip+Adam launch (SURVEY.md §8e).  Collection, GAE and advantage standardisation
are per-env-row and never cross ranks.  The reference has no counterpart (single learner; ray
actors only collect: manager/distributed_manager.py:7-65).

`critic_loss = max(mean1, mean2)` (ppo.py:151-154): the in-kernel exchange makes the two means GLOBAL (the ranks swap
their row sums right after the forward phase, csrc/ppo_fused.cu); only the NCCL fallback path (symmetric memory unavailable,
JB_NO_P2P=1, CNN heads) still evaluates the max per rank on its local minibatch shard.
"""
import torch
import torch.distributed as dist


P2P_FLAG_WORDS = 128 + 8 * 256 * 2     # JB_X_WORDS of include/jorldy_b200_fused.h (zeroed before the rendezvous)


def exchange_layout(num_flat, world_size):
    """Float offsets of the regions of one rank's exchange buffer (include/jorldy_b200_fused.h):
    gradient | owner inbox (LL words) | averaged gradient (LL words) | message words.  An LL word is 64 bits = 2 floats,
    written in 16-byte pairs: every region starts on a 32-byte boundary (jb_ppo_fused_run rejects anything else)."""
    if num_flat % 4:
        raise RuntimeError("flat parameter buffer is not a whole number of float4")
    q4 = (num_flat // 4 + world_size - 1) // world_size
    llin, llout = 8 * world_size * q4, 2 * num_flat
    llout += -llout % 8
    base = num_flat + (-num_flat % 8)
    return {"llin_off": base, "gred_off": base + llin, "flag_off": base + llin + llout,
            "n": base + llin + llout + P2P_FLAG_WORDS}


def _try_p2p(agent, world_size):
    """Peer-mapped gradient exchange buffer for the persistent PPO kernel (csrc/ppo_fused.cu): every rank's flat
    gradient lives in a symmetric-memory allocation whose peer pointers the kernel reads and writes over NVLink, so
    the gradient average (reduce-scatter by slice owners + all-gather by stores, flags in the same buffer) happens
    INSIDE the kernel instead of 6144 NCCL calls per learn().
    Falls back silently (agent.p2p = None -> CUDA graphs + NCCL) when symmetric memory is unavailable."""
    agent.p2p = None
    import os
    if os.environ.get("JB_NO_P2P", "0") == "1":          # operator override: CUDA graphs + ncclAllReduce instead
        return
    net = getattr(agent, "network", None)
    # (these conditions are identical on every rank, so the early return is itself a collective decision)
    if net is None or not net.flat.is_cuda or dist.get_backend() != "nccl" or world_size > 8 or type(agent).__name__ != "PPO":
        return
    # Step 1 — LOCAL probe only (no collective inside the try): can this rank allocate symmetric memory at all?
    ok, buf, hdl, ptrs, err = 1, None, None, None, None
    symm = None
    try:
        import torch.distributed._symmetric_memory as symm
        if net.num_flat % 4:
            raise RuntimeError("flat parameter buffer is not a whole number of float4")
        lay = exchange_layout(net.num_flat, world_size)
        n = lay["n"]
        buf = symm.empty(n, dtype=torch.float32, device=net.flat.device)
        buf.zero_()
        torch.cuda.synchronize()
    except Exception as e:      # pragma: no cover - depends on the platform
        ok, err = 0, e

    def agree(ok_local):
        flag = torch.tensor([ok_local], dtype=torch.int32, device=net.flat.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        return int(flag.item()) == 1

    def fallback():
        import warnings
        warnings.warn(f"in-kernel gradient exchange unavailable ({type(err).__name__ if err else 'peer'}: {err}); using NCCL all-reduce")

    # Step 2 — agree BEFORE the collective rendezvous: a rank that failed locally must not leave the others blocked in it
    if not agree(ok):
        return fallback()
    # Step 3 — the rendezvous itself is a collective every rank now enters; its outcome is agreed on again
    try:
        hdl = symm.rendezvous(buf, dist.group.WORLD)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        if len(ptrs) != world_size or ptrs[dist.get_rank()] != buf.data_ptr():
            raise RuntimeError("unexpected symmetric-memory pointer table")
    except Exception as e:      # pragma: no cover - depends on the platform
        ok, err = 0, e
    if not agree(ok):
        return fallback()
    net.rebind_grad(buf)
    dist.barrier()
    agent.p2p = {"buf": buf, "hdl": hdl, "ptrs": ptrs, "rank": dist.get_rank(), "world": world_size, "epoch": 0,
                 "llin_off": lay["llin_off"], "gred_off": lay["gred_off"], "flag_off": lay["flag_off"]}


def attach(agent, world_size, average_with="avg"):
    """Makes `agent` a data-parallel learner: identical initial weights on every rank (broadcast from
    rank 0) and an averaged flat gradient before every optimiser step."""
    if world_size <= 1:
        return agent
    if hasattr(agent, "critics") or getattr(agent, "replicas_only", False):
        # DDPG / TD3 / SAC (SURVEY 8f-4): several networks and optimisers per agent, no gradient exchange built for them;
        # V-MPO: its median and psi normalisation are per minibatch, so an averaged sharded gradient is another algorithm;
        # ICM-PPO: its BatchNorm batch statistics and its observation / intrinsic-reward running statistics are per replica.
        # Under torchrun every rank is an independent replica (own envs, own replay, own weights), and says so.
        import warnings
        family = agent.FAMILY if getattr(agent, "replicas_only", False) else "the actor-critic family"
        warnings.warn(f"{type(agent).__name__}: replicas only (no data-parallel learner for {family})")
        agent.world_size = 1
        return agent
    dist.broadcast(agent.network.flat, src=0)
    if hasattr(agent, "target_network"):
        dist.broadcast(agent.target_network.flat, src=0)
    agent.world_size = world_size

    def allreduce(flat_grad):
        if average_with == "avg":                       # NCCL: averaging fused into the collective
            dist.all_reduce(flat_grad, op=dist.ReduceOp.AVG)
        else:                                           # gloo (CPU tests) has no AVG
            dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
            flat_grad.div_(world_size)

    agent.allreduce = allreduce
    _try_p2p(agent, world_size)
    mem = getattr(agent, "memory", None)
    if mem is not None and hasattr(mem, "sample_device") and hasattr(mem, "tree_size"):
        mem.shard_world = world_size            # PER tree becomes one shard of a world_size-way replay
    return agent
