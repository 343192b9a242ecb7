"""Kernel-variant timing sweep (development tool, not the contract bench): times each scatter
variant with CUDA events on device-resident synthetic streams."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from event_utils_b200 import _lib  # noqa: E402

L = _lib.lib()
dev = torch.device("cuda")
HBM = 3350.0   # GB/s, H100 SXM data sheet (HBM3); a data-sheet figure, not a measurement


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = [ev[i].elapsed_time(ev[i + 1]) for i in range(iters)]
    return min(ts), sum(ts) / len(ts)


def uniform(n, H, W, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.rand(n, device=dev, generator=g) * (W - 1)
    y = torch.rand(n, device=dev, generator=g) * (H - 1)
    t = torch.sort(torch.rand(n, device=dev, generator=g)).values
    p = (torch.randint(0, 2, (n,), device=dev, generator=g) * 2 - 1).float()
    return x, y, t, p


def zipf(n, H, W, seed, s=1.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    npx = H * W
    w = 1.0 / torch.arange(1, npx + 1, device=dev, dtype=torch.float64) ** s
    cdf = torch.cumsum(w, 0) / w.sum()
    ranks = torch.searchsorted(cdf, torch.rand(n, device=dev, generator=g, dtype=torch.float64)).clamp_(max=npx - 1)
    perm = torch.randperm(npx, device=dev, generator=g)
    pix = perm[ranks]
    return (pix % W).float(), (pix // W).float()


def report(name, ms, n, bytes_per_event, extra_bytes=0):
    gbs = (n * bytes_per_event + extra_bytes) / ms / 1e6
    print("%-44s %8.3f ms  %9.1f Mev/s  %7.1f GB/s  %5.1f%% of %.0f" % (name, ms, n / ms / 1e3, gbs, 100 * gbs / HBM, HBM), flush=True)


N = int(os.environ.get("N", 50_000_000))
B, H, W = 5, 480, 640
x, y, t, p = uniform(N, H, W, 2024)
out = torch.empty((B, H, W), device=dev)
ws = torch.empty(L.evk_voxel_workspace_bytes(B, H, W, 0), dtype=torch.uint8, device=dev)
oob = torch.zeros(1, dtype=torch.int64, device=dev)
t0, dt = float(t[0]), float(t[-1] - t[0])
print("== voxel %d events -> %dx%dx%d" % (N, B, H, W))
ws = torch.empty(max(ws.numel(), L.evk_voxel_workspace_bytes(B, H, W, _lib.VARIANT_ROUTED)), dtype=torch.uint8, device=dev)
for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("vector_red", _lib.VARIANT_VECTOR_RED), ("routed", _lib.VARIANT_ROUTED)):
    def run(v=v, fl=0):
        _lib.check(L.evk_voxel_f32(x.data_ptr(), y.data_ptr(), t.data_ptr(), p.data_ptr(), N, t0, dt, B, H, W, v | fl,
                                   out.data_ptr(), ws.data_ptr(), ws.numel(), oob.data_ptr(), None))
    best, avg = timeit(run)
    report("voxel " + name, best, N, 16, 4 * B * H * W)
# the same stream with two hot pixels carrying 10 % of the events
xh, yh = x.clone(), y.clone()
hm = torch.rand(N, device=dev) < 0.10
xh[hm] = torch.where(torch.rand(int(hm.sum()), device=dev) < 0.5, 17.0, 400.0)
yh[hm] = torch.where(xh[hm] == 17.0, 33.0, 301.0)
for name, v in (("vector_red", _lib.VARIANT_VECTOR_RED), ("smem_cache", _lib.VARIANT_SMEM_TILE), ("routed", _lib.VARIANT_ROUTED), ("auto", 0)):
    for tag, (xx, yy) in (("uniform", (x, y)), ("10% hot pixels", (xh, yh))):
        def run(v=v, xx=xx, yy=yy):
            _lib.check(L.evk_voxel_f32(xx.data_ptr(), yy.data_ptr(), t.data_ptr(), p.data_ptr(), N, t0, dt, B, H, W, v,
                                       out.data_ptr(), ws.data_ptr(), ws.numel(), oob.data_ptr(), None))
        best, avg = timeit(run)
        report("voxel %s [%s]" % (name, tag), best, N, 16, 4 * B * H * W)
del xh, yh, hm
ev = torch.stack((x, y, t, p), 1).contiguous()
for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("vector_red", _lib.VARIANT_VECTOR_RED)):
    def run(v=v):
        _lib.check(L.evk_voxel_aos_f32(ev.data_ptr(), N, t0, dt, B, H, W, v, out.data_ptr(), ws.data_ptr(), ws.numel(), oob.data_ptr(), None))
    best, avg = timeit(run)
    report("voxel AoS " + name, best, N, 16, 4 * B * H * W)
del ev
out3 = torch.empty((B, H + 1, W + 1), device=dev)
ws3 = torch.empty(L.evk_voxel_workspace_bytes(B, H + 1, W + 1, _lib.BILINEAR), dtype=torch.uint8, device=dev)
for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("vector_red", _lib.VARIANT_VECTOR_RED)):
    def run(v=v):
        _lib.check(L.evk_voxel_f32(x.data_ptr(), y.data_ptr(), t.data_ptr(), p.data_ptr(), N, t0, dt, B, H + 1, W + 1,
                                   v | _lib.BILINEAR | _lib.CLIP, out3.data_ptr(), ws3.data_ptr(), ws3.numel(), oob.data_ptr(), None))
    best, avg = timeit(run)
    report("voxel trilinear " + name, best, N, 16, 4 * B * H * W)
# pure read baseline: how fast can 16 B/event be streamed at all (torch sum of the 4 arrays)
best, _ = timeit(lambda: (x.sum(), y.sum(), t.sum(), p.sum()))
report("(torch .sum() of the 4 arrays: read-only)", best, N, 16)

if os.environ.get("ONLY") == "voxel":
    sys.exit(0)
print("== event image %d events -> 720x1280" % N)
Hi, Wi = 720, 1280
for dist in ("uniform", "zipf1.0", "zipf1.2"):
    if dist == "uniform":
        xi, yi, _, pi = uniform(N, Hi, Wi, 99)
    else:
        xi, yi = zipf(N, Hi, Wi, 99, float(dist[4:]))
        pi = torch.ones(N, device=dev)
    img = torch.empty((Hi + 1, Wi + 1), device=dev)
    wsi = torch.empty(max(256, L.evk_image_workspace_bytes(Hi + 1, Wi + 1, _lib.BILINEAR)), dtype=torch.uint8, device=dev)
    for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("warp_agg", _lib.VARIANT_WARP_AGG), ("smem_cache", _lib.VARIANT_SMEM_TILE), ("auto", 0)):
        def run(v=v):
            _lib.check(L.evk_image_f32(xi.data_ptr(), yi.data_ptr(), pi.data_ptr(), N, Hi, Wi, 0.0, 0.0, v, 0.0, img.data_ptr(),
                                       wsi.data_ptr(), wsi.numel(), oob.data_ptr(), None))
        best, avg = timeit(run, iters=3, warm=1)
        report("image nearest %s %s" % (dist, name), best, N, 12, 4 * Hi * Wi)
    cnt = torch.empty((Hi, Wi), dtype=torch.int32, device=dev)
    for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("warp_agg", _lib.VARIANT_WARP_AGG), ("smem_cache", _lib.VARIANT_SMEM_TILE), ("auto", 0)):
        def run(v=v):
            _lib.check(L.evk_count_u32(xi.data_ptr(), yi.data_ptr(), N, Hi, Wi, 0.0, 0.0, v, cnt.data_ptr(), oob.data_ptr(), None))
        best, avg = timeit(run, iters=3, warm=1)
        report("count u32 %s %s" % (dist, name), best, N, 8, 4 * Hi * Wi)
    xb = xi + torch.rand(N, device=dev) * 0.999 if dist != "uniform" else xi
    yb = yi + torch.rand(N, device=dev) * 0.999 if dist != "uniform" else yi
    for name, v in (("global_red", _lib.VARIANT_GLOBAL_RED), ("vector_red", _lib.VARIANT_VECTOR_RED), ("smem_cache", _lib.VARIANT_SMEM_TILE)):
        def run(v=v):
            _lib.check(L.evk_image_f32(xb.data_ptr(), yb.data_ptr(), pi.data_ptr(), N, Hi + 1, Wi + 1, float(Wi), float(Hi),
                                       v | _lib.BILINEAR | _lib.CLIP, 0.0, img.data_ptr(), wsi.data_ptr(), wsi.numel(), oob.data_ptr(), None))
        best, avg = timeit(run, iters=3, warm=1)
        report("image bilinear %s %s" % (dist, name), best, N, 12, 4 * Hi * Wi)
    del xi, yi, pi, xb, yb
del x, y, t, p
torch.cuda.empty_cache()

print("== timestamp images, flow warp, neg/pos voxel (%d events)" % N)
xq, yq, tq, pq = uniform(N, 480, 640, 5)
tpos = torch.empty((481, 641), device=dev); tneg = torch.empty((481, 641), device=dev)
wst = torch.empty(L.evk_timestamp_image_workspace_bytes(481, 641), dtype=torch.uint8, device=dev)
best, _ = timeit(lambda: _lib.check(L.evk_timestamp_image_f32(xq.data_ptr(), yq.data_ptr(), tq.data_ptr(), pq.data_ptr(), N, float(tq[0]), float(tq[-1]),
                                                              481, 641, 640.0, 480.0, _lib.CLIP, tpos.data_ptr(), tneg.data_ptr(), wst.data_ptr(), wst.numel(),
                                                              oob.data_ptr(), None)), iters=3, warm=1)
report("timestamp images 480x640 (2 block REDs/event)", best, N, 16, 8 * 481 * 641)
flow = torch.randn(2, 480, 640, device=dev) * 20
xw, yw = torch.empty_like(xq), torch.empty_like(yq)
wsf = torch.empty(L.evk_warp_flow_workspace_bytes(480, 640), dtype=torch.uint8, device=dev)
for nm, wsp, wsb in (("planar flow", None, 0), ("interleaved flow", wsf.data_ptr(), wsf.numel())):
    best, _ = timeit(lambda: _lib.check(L.evk_warp_flow_f32(xq.data_ptr(), yq.data_ptr(), tq.data_ptr(), N, flow.data_ptr(), 480, 640, float(tq[-1]),
                                                            xw.data_ptr(), yw.data_ptr(), wsp, wsb, None)), iters=3, warm=1)
    report("dense-flow warp 480x640, %s" % nm, best, N, 20)
outnp = torch.empty((2, 5, 480, 640), device=dev)
wsnp = torch.empty(2 * L.evk_voxel_workspace_bytes(5, 480, 640, 0), dtype=torch.uint8, device=dev)
best, _ = timeit(lambda: _lib.check(L.evk_voxel_negpos_f32(xq.data_ptr(), yq.data_ptr(), tq.data_ptr(), pq.data_ptr(), N, 0.0, 1.0, 5, 480, 640,
                                                           _lib.AUTO_SPAN, outnp.data_ptr(), wsnp.data_ptr(), wsnp.numel(), oob.data_ptr(), None)), iters=3, warm=1)
report("neg/pos voxel 2x5x480x640, one pass", best, N, 16, 8 * 5 * 480 * 640)
del xq, yq, tq, pq, xw, yw, flow
torch.cuda.empty_cache()

print("== cmax %d events (f64 parity mode / f32 fast mode)" % N)
g = torch.Generator(device=dev).manual_seed(7)
for scene in ("uniform", "lattice"):
    t64 = torch.sort(torch.rand(N, device=dev, generator=g, dtype=torch.float64)).values * 0.05
    if scene == "uniform":
        x64 = torch.rand(N, device=dev, generator=g, dtype=torch.float64) * 239
        y64 = torch.rand(N, device=dev, generator=g, dtype=torch.float64) * 179
    else:
        k = torch.randint(1, 11, (N,), device=dev, generator=g).double() * 20
        along = torch.rand(N, device=dev, generator=g, dtype=torch.float64)
        vert = torch.rand(N, device=dev, generator=g) < 0.5
        x64 = torch.where(vert, k, along * 239) + (t64 - t64[-1]) * 60.0
        y64 = torch.where(vert, along * 179, k.clamp(max=170)) + (t64 - t64[-1]) * -35.0
    p64 = torch.ones(N, device=dev, dtype=torch.float64)
    wsc = torch.empty(L.evk_cmax_workspace_bytes(180, 240), dtype=torch.uint8, device=dev)
    res = torch.empty(8, dtype=torch.float64, device=dev)
    tl = float(t64[-1])
    for params in ((45.0, -20.0), (60.0, -35.0)):
        for fl, nm in ((_lib.CMAX_WANT_GRAD, "f+g"), (0, "f")):
            def run(fl=fl, params=params):
                _lib.check(L.evk_cmax_linvel_variance_f64(x64.data_ptr(), y64.data_ptr(), t64.data_ptr(), p64.data_ptr(), N, 1.0,
                                                          params[0], params[1], tl, 180, 240, 180, 240, 1.0, fl, res.data_ptr(),
                                                          None, None, wsc.data_ptr(), wsc.numel(), None))
            best, avg = timeit(run, iters=3, warm=1)
            report("cmax f64 %s %s v=%s" % (scene, nm, params), best, N, 32)
    x32, y32, p32 = x64.float(), y64.float(), p64.float()
    t32 = (t64 - tl).float()
    def run32():
        _lib.check(L.evk_cmax_linvel_variance_f32(x32.data_ptr(), y32.data_ptr(), t32.data_ptr(), p32.data_ptr(), N, 1.0, 45.0, -20.0,
                                                  180, 240, 180, 240, 1.0, _lib.CMAX_WANT_GRAD, res.data_ptr(), None, None,
                                                  wsc.data_ptr(), wsc.numel(), None))
    best, avg = timeit(run32, iters=3, warm=1)
    report("cmax f32 %s f+g" % scene, best, N, 16)
    if scene == "uniform":
        flow_c = torch.randn(2, 180, 240, device=dev) * 30
        tf = (t64).float()
        def runflow():
            _lib.check(L.evk_cmax_flow_variance_f32(x32.data_ptr(), y32.data_ptr(), tf.data_ptr(), p32.data_ptr(), N, flow_c.data_ptr(), float(tf[-1]),
                                                    180, 240, 1.0, 0, res.data_ptr(), None, wsc.data_ptr(), wsc.numel(), None))
        best, avg = timeit(runflow, iters=3, warm=1)
        report("cmax dense-flow warp + IWE + variance (f only)", best, N, 16)
        del flow_c, tf
    print("   result", res.cpu().numpy())
    del x64, y64, t64, p64, x32, y32, t32, p32
