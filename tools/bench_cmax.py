"""Timing of one full contrast-maximisation evaluation (memset + event pass + tail) per event-pass back end:
"l2" = block accumulator in L2 (vector reductions), "onchip" = IWE in shared memory (cmax_onchip_kernel).
Development tool; CUDA events, device-resident streams."""
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


def report(name, ms, n, bpe):
    gbs = n * bpe / ms / 1e6
    print("%-58s %8.3f ms  %9.1f Mev/s  %7.1f GB/s  %5.1f%% of %.0f" % (name, ms, n / ms / 1e3, gbs, 100 * gbs / HBM, HBM), flush=True)


sizes = [int(v) for v in os.environ.get("SIZES", "50000000").split(",")]
BACKENDS = (("l2", _lib.VARIANT_VECTOR_RED), ("onchip", _lib.VARIANT_SMEM_TILE))
for N in sizes:
    print("== cmax %d events" % N)
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
            del k, along, vert
        p64 = (torch.randint(0, 2, (N,), device=dev, generator=g) * 2 - 1).double()
        wsc = torch.empty(L.evk_cmax_workspace_bytes(180, 240), dtype=torch.uint8, device=dev)
        res = torch.empty(12, dtype=torch.float64, device=dev)
        tl = float(t64[-1])
        params = (60.0, -35.0)      # the lattice scene's true motion: sharpest image, worst same-address contention
        for bname, bflag in BACKENDS:
            for fl, nm in ((_lib.CMAX_WANT_GRAD, "f+g"), (0, "f")):
                def run(fl=fl):
                    _lib.check(L.evk_cmax_linvel_variance_f64(x64.data_ptr(), y64.data_ptr(), t64.data_ptr(), p64.data_ptr(), N, 1.0,
                                                              params[0], params[1], tl, 180, 240, 180, 240, 1.0, fl | bflag, res.data_ptr(),
                                                              None, None, wsc.data_ptr(), wsc.numel(), None))
                best, avg = timeit(run, iters=4, warm=1)
                report("cmax f64 %-7s %-6s %-3s (f=%.6g)" % (scene, bname, nm, res[0].item()), best, N, 32)
        x32, y32, p32 = x64.float(), y64.float(), p64.float()
        t32 = (t64 - tl).float()
        del x64, y64, t64, p64
        for bname, bflag in BACKENDS:
            for fl, nm in ((_lib.CMAX_WANT_GRAD, "f+g"), (0, "f")):
                def run32(fl=fl):
                    _lib.check(L.evk_cmax_linvel_variance_f32(x32.data_ptr(), y32.data_ptr(), t32.data_ptr(), p32.data_ptr(), N, 1.0, params[0], params[1],
                                                              180, 240, 180, 240, 1.0, fl | bflag, res.data_ptr(), None, None,
                                                              wsc.data_ptr(), wsc.numel(), None))
                best, avg = timeit(run32, iters=4, warm=1)
                report("cmax f32 %-7s %-6s %-3s (f=%.6g)" % (scene, bname, nm, res[0].item()), best, N, 16)
        if scene == "uniform":
            flow_c = torch.randn(2, 180, 240, device=dev) * 30
            tf = t32 + tl
            for bname, bflag in BACKENDS:
                def runflow():
                    _lib.check(L.evk_cmax_flow_variance_f32(x32.data_ptr(), y32.data_ptr(), tf.data_ptr(), p32.data_ptr(), N, flow_c.data_ptr(), float(tl),
                                                            180, 240, 1.0, bflag, res.data_ptr(), None, wsc.data_ptr(), wsc.numel(), None))
                best, avg = timeit(runflow, iters=3, warm=1)
                report("cmax dense-flow warp + IWE + variance %-6s (f only)" % bname, best, N, 16)
            del flow_c, tf
        del x32, y32, t32, p32
        torch.cuda.empty_cache()
