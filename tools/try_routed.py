"""Development driver for the routed voxel kernel: parity vs the oracle at growing sizes, then timing."""
import os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from event_utils_b200 import _lib
from oracle import evk_oracle as O
L = _lib.lib()
B, H, W = 5, 480, 640
def run(x, y, t, p, variant, B=B, H=H, W=W, reps=1):
    n = x.shape[0]
    out = torch.empty((B, H, W), device="cuda")
    ws = torch.empty(L.evk_voxel_workspace_bytes(B, H, W, variant), dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    t0, dt = float(t[0]), float(t[-1] - t[0])
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(L.evk_voxel_f32(x.data_ptr(), y.data_ptr(), t.data_ptr(), p.data_ptr(), n, t0, dt, B, H, W, variant,
                                   out.data_ptr(), ws.data_ptr(), ws.numel(), oob.data_ptr(), None))
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return out, min(ts), int(oob.item())
for n, (h, w) in ((1000, (4, 6)), (5000, (48, 64)), (100000, (260, 346)), (1_000_003, (480, 640)), (8_000_000, (480, 640))):
    rng = np.random.default_rng(n)
    x = (rng.random(n) * (w - 1)).astype(np.float32); y = (rng.random(n) * (h - 1)).astype(np.float32)
    t = np.sort(rng.random(n)).astype(np.float32); p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    if n == 100000:
        p[::7] = 0.5; p[::11] = 0.0; x[5] = -1.0     # slow-path events, a wrapped coordinate
    ref = O.voxel_f32(x, y, t, p, B, (h, w))
    X, Y, T, P = (torch.from_numpy(a).cuda() for a in (x, y, t, p))
    out, ms, oob = run(X, Y, T, P, _lib.VARIANT_ROUTED, H=h, W=w)
    err = float(np.abs(out.cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-30))
    print("n=%d %dx%d routed: max rel err %.3e oob %d  %.3f ms" % (n, h, w, err, oob, ms), flush=True)
    # unaligned views (head peel)
    if n > 5000:
        out2, _, _ = run(X[1:], Y[1:], T[1:], P[1:], _lib.VARIANT_ROUTED, H=h, W=w)
        ref2 = O.voxel_f32(x[1:], y[1:], t[1:], p[1:], B, (h, w))
        print("   offset-by-one views: max rel err %.3e" % float(np.abs(out2.cpu().numpy() - ref2).max() / np.abs(ref2).max()), flush=True)
N = 50_000_000
g = torch.Generator(device="cuda").manual_seed(2024)
x = torch.rand(N, device="cuda", generator=g) * 639; y = torch.rand(N, device="cuda", generator=g) * 479
t = torch.sort(torch.rand(N, device="cuda", generator=g)).values; p = (torch.randint(0, 2, (N,), device="cuda", generator=g) * 2 - 1).float()
for name, v in (("vector_red", _lib.VARIANT_VECTOR_RED), ("routed", _lib.VARIANT_ROUTED)):
    out, ms, oob = run(x, y, t, p, v, reps=5)
    print("%s 50M: %.3f ms  (%.1f%% of 3350 GB/s) sum=%.1f" % (name, ms, 100 * (16 * N + 4 * B * H * W) / ms / 1e6 / 3350.0, float(out.double().sum())), flush=True)
    if name == "vector_red": base = out.clone()
print("50M routed vs vector_red: max rel diff %.3e" % float((out - base).abs().max() / base.abs().max()))
