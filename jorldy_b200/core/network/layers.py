"""Thin python wrappers over the C-ABI dense kernels (argument marshalling only)."""
from ..dev import C, ptr, stream_ptr


import os

TC_MIN_ROWS = 1024     # below this a 128x128 tile grid cannot fill the 132 SMs: stay on the fp32 FFMA tiles
_USE_TC = os.environ.get("JB_NO_TC", "0") != "1"


def linear_fwd(x, w, b, y, relu):
    """y = act(x W^T + b).  Large-M products (env-row batches) go to the wgmma 3xTF32 kernel
    (csrc/tc_gemm.cu); minibatch-sized ones to the fp32 FFMA tiles (csrc/linear.cu)."""
    M, in_f = x.shape
    out_f = w.shape[0]
    if _USE_TC and M >= TC_MIN_ROWS and M % 128 == 0 and out_f % 128 == 0 and in_f % 32 == 0 and b is not None:
        C.jb_linear_fwd_tc(ptr(x), ptr(w), ptr(b), ptr(y), M, in_f, out_f, int(relu), stream_ptr())
        return
    C.jb_linear_fwd(ptr(x), ptr(w), ptr(b), ptr(y), M, in_f, out_f, int(relu), stream_ptr())


def linear_bwd_dx(dy, w, dx, relu_act=None, accumulate=False):
    M, out_f = dy.shape
    in_f = w.shape[1]
    if accumulate:
        C.jb_gemm(ptr(dy), out_f, 1, ptr(w), in_f, 0, ptr(dx), in_f, M, in_f, out_f, 0, 0,
                  ptr(relu_act), in_f, 0, 1, stream_ptr())
    else:
        C.jb_linear_bwd_dx(ptr(dy), ptr(w), ptr(dx), M, in_f, out_f, ptr(relu_act), stream_ptr())


def linear_bwd_dw(dy, x, dw, db):
    M, out_f = dy.shape
    C.jb_linear_bwd_dw(ptr(dy), ptr(x), ptr(dw), ptr(db), M, x.shape[1], out_f, stream_ptr())


def linear_io_fwd(x, w, b, y, relu):
    M, in_f = x.shape
    C.jb_linear_io_fwd(ptr(x), ptr(w), ptr(b), ptr(y), M, in_f, w.shape[1], int(relu), stream_ptr())


def linear_io_bwd_dx(dy, w, dx, relu_act=None, accumulate=False):
    M, out_f = dy.shape
    in_f = w.shape[0]
    if accumulate:
        C.jb_gemm(ptr(dy), out_f, 1, ptr(w), out_f, 1, ptr(dx), in_f, M, in_f, out_f, 0, 0,
                  ptr(relu_act), in_f, 0, 1, stream_ptr())
    else:
        C.jb_linear_io_bwd_dx(ptr(dy), ptr(w), ptr(dx), M, in_f, out_f, ptr(relu_act), stream_ptr())


def linear_io_bwd_dw(dy, x, dw, db):
    M, out_f = dy.shape
    C.jb_linear_io_bwd_dw(ptr(dy), ptr(x), ptr(dw), M, x.shape[1], out_f, stream_ptr())
    C.jb_colsum(ptr(dy), M, out_f, ptr(db), 0, stream_ptr())


def heads_fwd(h, heads, out):
    """heads: list of up to 3 (w, b) pairs, w [n,H]."""
    M, H = h.shape
    a = []
    for i in range(3):
        if i < len(heads):
            w, b = heads[i]
            a += [ptr(w), ptr(b), w.shape[0]]
        else:
            a += [0, 0, 0]
    C.jb_heads_fwd(ptr(h), M, H, *a, ptr(out), stream_ptr())


def heads_bwd_dx(dout, h, heads, dh):
    M, H = h.shape
    a = []
    for i in range(3):
        if i < len(heads):
            a += [ptr(heads[i][0]), heads[i][0].shape[0]]
        else:
            a += [0, 0]
    C.jb_heads_bwd_dx(ptr(dout), ptr(h), M, H, *a, ptr(dh), stream_ptr())


def heads_bwd_dw(dout, h, grads):
    """grads: list of up to 3 (dw, db) pairs."""
    M, H = h.shape
    a = []
    for i in range(3):
        if i < len(grads):
            dw, db = grads[i]
            a += [ptr(dw), ptr(db), dw.shape[0]]
        else:
            a += [0, 0, 0]
    C.jb_heads_bwd_dw(ptr(dout), ptr(h), M, H, *a, stream_ptr())
