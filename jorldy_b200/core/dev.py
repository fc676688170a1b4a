"""Device plumbing shared by the host-side classes: torch owns memory and streams, the C ABI
gets raw pointers."""
import torch

from .._lib import C, JbError  # noqa: F401


def stream_ptr():
    """cudaStream_t of torch's current stream (the capture stream under CUDA-graph capture)."""
    return torch.cuda.current_stream().cuda_stream


def capture_after_warmup(fn, restore=(), repeat=1):
    """A CUDA graph of `repeat` calls of fn().  fn() first runs once eagerly on a side stream, which allocates its
    workspaces; the tensors in `restore` then get back the values they had before it.  Capture does not execute."""
    saved = [t.clone() for t in restore]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for dst, src in zip(restore, saved):
        dst.copy_(src)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(repeat):
            fn()
    return graph


def ptr(t):
    return 0 if t is None else t.data_ptr()


def require_cuda(device):
    device = torch.device(device) if device is not None else torch.device("cuda")
    if device.type != "cuda":
        raise JbError(
            f"jorldy_b200 runs its hot path only on CUDA (sm_90a); got device '{device}'. "
            "There is no CPU fallback — use the reference (or oracle/) for CPU runs.")
    if not torch.cuda.is_available():
        raise JbError("CUDA is not available: jorldy_b200 has no CPU fallback.")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def f32(x, device):
    """as_tensor(float32) on the device (jorldy/core/agent/base.py:61-73)."""
    return torch.as_tensor(x, dtype=torch.float32, device=device)
