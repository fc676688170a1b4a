"""Host side of the persistent PPO minibatch-loop kernel (csrc/ppo_fused.cu): builds the
jb_ppo_fused_args block (include/jorldy_b200_fused.h) from the agent's tensors."""
import ctypes

import torch

from ..dev import C, ptr, stream_ptr

_P = ctypes.c_void_p


class FusedArgs(ctypes.Structure):
    _fields_ = [
        ("W1", _P), ("b1", _P), ("W2", _P), ("b2", _P), ("Wh", _P * 3), ("bh", _P * 3),
        ("gW1", _P), ("gb1", _P), ("gW2", _P), ("gb2", _P), ("gWh", _P * 3), ("gbh", _P * 3),
        ("flat", _P), ("grad", _P), ("am", _P), ("av", _P), ("P4", ctypes.c_longlong),
        ("state", _P), ("action", _P), ("adv", _P), ("ret", _P), ("vold", _P), ("logp_old", _P), ("perm", _P),
        ("h1", _P), ("h2", _P), ("xg", _P), ("w1p", _P), ("headp", _P),
        ("dout", _P), ("dv2", _P), ("rowst", _P), ("h2t", _P), ("W2t", _P), ("W2img", _P), ("W2Timg", _P), ("partials", _P), ("acc", _P),
        ("cur_idx", _P), ("barrier", _P), ("step", _P), ("cursor", _P), ("lr", _P),
        ("peer", _P * 8), ("world", ctypes.c_int), ("rank", ctypes.c_int), ("xbase", ctypes.c_uint), ("xflag_off", ctypes.c_int), ("xgred_off", ctypes.c_int), ("xllin_off", ctypes.c_int),
        ("nh", ctypes.c_int * 3),
        ("B", ctypes.c_int), ("D", ctypes.c_int), ("H", ctypes.c_int), ("A", ctypes.c_int), ("nout", ctypes.c_int),
        ("continuous", ctypes.c_int), ("n_steps", ctypes.c_int),
        ("eps_clip", ctypes.c_float), ("vf_coef", ctypes.c_float), ("ent_coef", ctypes.c_float),
        ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("adam_eps", ctypes.c_float), ("max_norm", ctypes.c_float),
    ]


def supported(agent, B):
    net = agent.network
    head = getattr(net, "head", None)
    return (getattr(head, "kind", None) == "mlp" and type(agent.optimizer).__name__ == "Adam"
            and (agent.allreduce is None or getattr(agent, "p2p", None) is not None)
            and B % 32 == 0 and B <= 512 and net.D_hidden % 32 == 0 and net.D_hidden <= 512 and head.D_in <= 16 and net.nout <= 8
            and head.D_head_out == net.D_hidden and agent.action_size <= 8)


class FusedRunner:
    def __init__(self, agent, B):
        assert ctypes.sizeof(FusedArgs) == C.jb_ppo_fused_args_size(), "jb_ppo_fused_args layout mismatch"
        self.agent, self.B = agent, B
        net, dev = agent.network, agent.device
        H, D = net.D_hidden, net.head.D_in
        self.ws = {
            "h1": torch.empty(B, H, device=dev), "h2": torch.empty(B, H, device=dev), "xg": torch.empty(B, D, device=dev),
            "w1p": torch.zeros(B // 32, H, D + 1, device=dev), "headp": torch.zeros(H // 32, 2, B, 4, device=dev),
            "dout": torch.zeros(B, 8, device=dev), "dv2": torch.zeros(B, device=dev), "rowst": torch.zeros(6, B, device=dev),
            "h2t": torch.empty(H // 32, B, 32, device=dev), "W2t": torch.empty(H // 32, H, 32, device=dev),
            "W2img": torch.empty(2, H // 32, H // 32, 1024, device=dev),
            "W2Timg": torch.empty(2, max(H // 128, 1), H // 32, 4096, device=dev),
            "partials": torch.zeros(256, device=dev), "cur_idx": torch.zeros(B, dtype=torch.int32, device=dev),
            "barrier": torch.zeros(64, dtype=torch.int32, device=dev),
        }
        self.max_ctas = C.jb_ppo_fused_max_ctas()
        self.n_runs = 0

    def run(self, st, n_steps):
        ag = self.agent
        net, opt = ag.network, ag.optimizer
        opt._sync_lr()
        a = FusedArgs()
        p, g = net.p, net.g
        a.W1, a.b1, a.W2, a.b2 = ptr(p["head.l.weight"]), ptr(p["head.l.bias"]), ptr(p["l.weight"]), ptr(p["l.bias"])
        a.gW1, a.gb1, a.gW2, a.gb2 = ptr(g["head.l.weight"]), ptr(g["head.l.bias"]), ptr(g["l.weight"]), ptr(g["l.bias"])
        for i in range(3):
            if i < len(net.out_heads):
                n = net.out_heads[i][0]
                a.Wh[i], a.bh[i] = ptr(p[f"{n}.weight"]), ptr(p[f"{n}.bias"])
                a.gWh[i], a.gbh[i] = ptr(g[f"{n}.weight"]), ptr(g[f"{n}.bias"])
                a.nh[i] = net.out_heads[i][1]
            else:
                a.Wh[i] = a.bh[i] = a.gWh[i] = a.gbh[i] = None
                a.nh[i] = 0
        a.flat, a.grad, a.am, a.av = ptr(net.flat), ptr(net.grad), ptr(opt.exp_avg), ptr(opt.exp_avg_sq)
        a.P4 = net.num_flat // 4
        a.state, a.action = ptr(st["state"]), ptr(st["action"])
        a.adv, a.ret, a.vold, a.logp_old, a.perm = ptr(st["adv"]), ptr(st["ret"]), ptr(st["value"]), ptr(st["logp_old"]), ptr(st["perm"])
        ws = self.ws
        a.h1, a.h2, a.xg, a.w1p, a.headp = ptr(ws["h1"]), ptr(ws["h2"]), ptr(ws["xg"]), ptr(ws["w1p"]), ptr(ws["headp"])
        a.dout, a.dv2, a.rowst = ptr(ws["dout"]), ptr(ws["dv2"]), ptr(ws["rowst"])
        a.h2t, a.W2t, a.W2img, a.W2Timg = ptr(ws["h2t"]), ptr(ws["W2t"]), ptr(ws["W2img"]), ptr(ws["W2Timg"])
        a.partials, a.acc, a.cur_idx, a.barrier = ptr(ws["partials"]), ptr(ag._acc), ptr(ws["cur_idx"]), ptr(ws["barrier"])
        a.step, a.cursor, a.lr = ptr(opt._step_dev), ptr(ag._cursor), ptr(opt._lr_dev)
        a.B, a.D, a.H, a.A, a.nout = self.B, net.head.D_in, net.D_hidden, ag.action_size, net.nout
        a.continuous, a.n_steps = int(ag.continuous), int(n_steps)
        a.eps_clip, a.vf_coef, a.ent_coef = ag.epsilon_clip, ag.vf_coef, ag.ent_coef
        a.beta1, a.beta2, a.adam_eps = opt.betas[0], opt.betas[1], opt.eps
        a.max_norm = float(ag.clip_grad_norm) if ag.clip_grad_norm else 0.0
        p2p = getattr(ag, "p2p", None)
        if p2p is not None and self.n_runs < 4:
            # The kernel spins on flags written by the peers' kernels.  During the first launches the ranks' hosts are
            # still far apart (lazy allocations, CUDA-graph capture of the collect loop, module loading), and a host
            # call that has to wait for a peer DEVICE while that device spins on this rank's not-yet-launched kernel
            # would deadlock until the kernel's time-out: meet on the host with idle GPUs, then launch at once.
            import torch.distributed as dist
            torch.cuda.synchronize()
            dist.barrier()
            torch.cuda.synchronize()
        self.n_runs += 1
        if p2p is not None:
            assert net.grad.data_ptr() == p2p["ptrs"][p2p["rank"]], "gradient buffer is not the peer-mapped exchange buffer"
            for r in range(8):
                a.peer[r] = p2p["ptrs"][r] if r < p2p["world"] else None
            a.world, a.rank, a.xbase, a.xflag_off = p2p["world"], p2p["rank"], p2p["epoch"] & 0xFFFFFFFF, p2p["flag_off"]
            a.xgred_off, a.xllin_off = p2p["gred_off"], p2p["llin_off"]
            p2p["epoch"] += int(n_steps)
        else:
            a.world, a.rank, a.xbase, a.xflag_off, a.xgred_off, a.xllin_off = 1, 0, 0, 0, 0, 0
        C.jb_ppo_fused_run(ctypes.addressof(a), stream_ptr())
