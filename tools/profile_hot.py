"""ncu target: the hot-spot image kernel on Zipf(1.0) and Zipf(1.2) streams, nearest and bilinear (run under
`ncu -k regex:image_hot` by tools/gpu/bundle_ncu.sh, or stand-alone for CUDA-event timings)."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from event_utils_b200 import _lib
L = _lib.lib()
dev = torch.device("cuda")
N, H, W = 50_000_000, 720, 1280
g = torch.Generator(device=dev).manual_seed(99)
npx = H * W
img = torch.empty((H + 1, W + 1), device=dev)
ws = torch.empty(L.evk_image_workspace_bytes(H + 1, W + 1, _lib.BILINEAR), dtype=torch.uint8, device=dev)
oob = torch.zeros(1, dtype=torch.int64, device=dev)
for s_exp in (1.0, 1.2):
    w = 1.0 / torch.arange(1, npx + 1, device=dev, dtype=torch.float64) ** s_exp
    cdf = torch.cumsum(w, 0) / w.sum()
    ranks = torch.searchsorted(cdf, torch.rand(N, device=dev, generator=g, dtype=torch.float64)).clamp_(max=npx - 1)
    pix = torch.randperm(npx, device=dev, generator=g)[ranks]
    x, y = (pix % W).float(), (pix // W).float()
    p = torch.ones(N, device=dev)
    xb, yb = x + torch.rand(N, device=dev) * 0.999, y + torch.rand(N, device=dev) * 0.999
    del w, cdf, ranks, pix
    for name, fn in (("nearest", lambda: L.evk_image_f32(x.data_ptr(), y.data_ptr(), p.data_ptr(), N, H, W, 0.0, 0.0, 0, 0.0, img.data_ptr(), None, 0, oob.data_ptr(), None)),
                     ("bilinear", lambda: L.evk_image_f32(xb.data_ptr(), yb.data_ptr(), p.data_ptr(), N, H + 1, W + 1, float(W), float(H), _lib.BILINEAR | _lib.CLIP, 0.0,
                                                          img.data_ptr(), ws.data_ptr(), ws.numel(), oob.data_ptr(), None))):
        ts = []
        for _ in range(4):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); _lib.check(fn()); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = min(ts[1:])
        print("zipf s=%.1f %-8s auto: %.3f ms  %.1f%% of 3350 GB/s (12 B/event)" % (s_exp, name, ms, 100 * 12.0 * N / ms / 1e6 / 3350.0), flush=True)
    del x, y, p, xb, yb
