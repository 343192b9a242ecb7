"""Argument normalisation shared by the drop-in functions (host-side plumbing only)."""
import numpy as np
import torch

from .. import _lib, config


def variant_flag():
    v = config.variant
    if v is None:
        return _lib.VARIANT_AUTO
    return {"global_red": _lib.VARIANT_GLOBAL_RED, "vector_red": _lib.VARIANT_VECTOR_RED,
            "warp_agg": _lib.VARIANT_WARP_AGG, "routed": _lib.VARIANT_ROUTED, "smem_cache": _lib.VARIANT_SMEM_TILE, "auto": _lib.VARIANT_AUTO}[v]


def as_tensor(a):
    if isinstance(a, torch.Tensor):
        return a
    return torch.from_numpy(np.ascontiguousarray(a))


def needs_grad(*inputs):
    """True when autograd has to record the call: grad mode is on and one of the differentiable inputs requires grad."""
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs)


def compute_device(*tensors):
    """CUDA device the kernels run on: the inputs' device, or the default one for host inputs."""
    for t in tensors:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    d = torch.device(config.default_device)
    if d.index is None:
        d = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
    return d


def to_device(t, dev):
    """A tensor on `dev`: large host tensors through the library's upload path (_lib.upload), the rest through torch."""
    if t.is_cuda or t.numel() * t.element_size() < _lib.UPLOAD_MIN_BYTES:
        return t.to(dev, non_blocking=True)
    return _lib.upload([t.contiguous()], dev)[0]


def coords_f32(c, dev):
    """Event coordinates as contiguous f32 on `dev` with the reference's `.long()` semantics kept:
    f32 goes to the kernel untouched (it truncates); other float types are truncated first so
    that rounding to f32 cannot cross an integer; integers are exact in f32 below 2^24."""
    c = as_tensor(c).reshape(-1)
    if c.dtype == torch.float32:
        return to_device(c, dev).contiguous()
    c = to_device(c, dev)
    if c.dtype.is_floating_point:
        c = c.long()
    if c.dtype in (torch.int64, torch.int32):
        c = c.clamp(-(1 << 24), 1 << 24)   # anything beyond is out of range for any sensor, and stays so
    return c.to(torch.float32).contiguous()


def weights_f32(p, dev):
    p = to_device(as_tensor(p).reshape(-1), dev)
    return p.to(torch.float32).contiguous()


def aos_base(xs, ys, ts, ps):
    """If the four arrays are the columns [x,y,t,p] of one contiguous (N,4) f32 tensor
    (the data-loader layout, base_dataset.py:306,510) return a view of it, else None."""
    ts_ = (xs, ys, ts, ps)
    if not all(isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.dim() == 1 for t in ts_):
        return None
    n = xs.shape[0]
    if n == 0 or any(t.shape[0] != n for t in ts_):
        return None
    if n > 1 and any(t.stride(0) != 4 for t in ts_):
        return None
    base_ptr = xs.untyped_storage().data_ptr()
    if any(t.untyped_storage().data_ptr() != base_ptr for t in ts_):
        return None
    o = xs.storage_offset()
    if [t.storage_offset() for t in ts_] != [o, o + 1, o + 2, o + 3]:
        return None
    if xs.data_ptr() % 16 != 0:
        return None
    return torch.as_strided(xs, (n, 4), (4, 1))


def raise_if_oob(counter, what, shape):
    """Reproduce the reference's IndexError (image.py:96-99) from the device counter."""
    if not config.check_index_errors:
        return
    bad = int(counter.item())
    if bad:
        raise IndexError("%d events index outside the %s of shape %s" % (bad, what, tuple(shape)))
