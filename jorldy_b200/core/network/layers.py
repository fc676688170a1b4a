"""Thin python wrappers over the C-ABI dense kernels (argument marshalling only)."""
from ..dev import C, ptr, stream_ptr


import ctypes
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


def _ptrs(ts, kind=ctypes.c_void_p):
    return (kind * len(ts))(*ts)


def heads_fwd(h, heads, out):
    """heads: list of up to 4 (w, b) pairs, w [n,H]."""
    M, H = h.shape
    C.jb_heads_fwd_n(ptr(h), M, H, len(heads), _ptrs([ptr(w) for w, _ in heads]), _ptrs([ptr(b) for _, b in heads]),
                     _ptrs([w.shape[0] for w, _ in heads], ctypes.c_int), ptr(out), stream_ptr())


def heads_bwd_dx(dout, h, heads, dh):
    M, H = h.shape
    C.jb_heads_bwd_dx_n(ptr(dout), ptr(h), M, H, len(heads), _ptrs([ptr(w) for w, _ in heads]),
                        _ptrs([w.shape[0] for w, _ in heads], ctypes.c_int), ptr(dh), stream_ptr())


def heads_bwd_dw(dout, h, grads):
    """grads: list of up to 4 (dw, db) pairs."""
    M, H = h.shape
    C.jb_heads_bwd_dw_n(ptr(dout), ptr(h), M, H, len(grads), _ptrs([ptr(dw) for dw, _ in grads]),
                        _ptrs([ptr(db) for _, db in grads]), _ptrs([dw.shape[0] for dw, _ in grads], ctypes.c_int),
                        stream_ptr())
