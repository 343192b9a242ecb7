"""Timing of the rotation / 4-DoF contrast-maximisation evaluations (evk_cmax_warp_objective_*) next to linvel's, at
1 M and 50 M device-resident events: f only, f + g, the gradient pass alone (cmax_grad_pass_kernel, from
torch.profiler in a separate run) and a 32-model batch (f only).  Each figure is printed with its byte floor -- the
event bytes the evaluation must read over the data sheet's HBM bandwidth.

  python tools/bench_cmax_warps.py [--sizes 1000000,50000000] [--baseline-lib PATH] [--out DIR]

--baseline-lib: another build of libevk.so (e.g. of the parent commit); its linvel f and f + g are timed alternately
with this build's, in the same process, to compare them within run-to-run spread.  Development tool."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from event_utils_b200 import _lib  # noqa: E402

HBM = 3.35e12   # B/s, H100 SXM data sheet (HBM3); a data-sheet figure, not a measurement


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
    return min(ev[i].elapsed_time(ev[i + 1]) for i in range(iters))


def kernel_ms(fn, name, iters=5):
    """mean device time of the kernels whose name contains `name`, per call of fn (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if name in e.key:
            total += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    return total / iters / 1e3


def declare_linvel(L):
    vp, i64, f32, f64, ci, cu, sz = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_int, ctypes.c_uint, ctypes.c_size_t
    L.evk_cmax_workspace_bytes.restype, L.evk_cmax_workspace_bytes.argtypes = sz, [ci, ci]
    L.evk_cmax_linvel_variance_f64.restype = ci
    L.evk_cmax_linvel_variance_f64.argtypes = [vp, vp, vp, vp, i64, f64, f64, f64, f64, ci, ci, ci, ci, f64, cu, vp, vp, vp, vp, sz, vp]
    L.evk_cmax_linvel_variance_f32.restype = ci
    L.evk_cmax_linvel_variance_f32.argtypes = [vp, vp, vp, vp, i64, f32, f32, f32, ci, ci, ci, ci, f64, cu, vp, vp, vp, vp, sz, vp]
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,50000000")
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = _lib.lib()
    base = declare_linvel(ctypes.CDLL(a.baseline_lib)) if a.baseline_lib else None
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name()
    print("card: %s" % card, flush=True)
    rows = []

    def report(what, ms, floor_bytes):
        floor = floor_bytes / HBM * 1e3
        rows.append({"what": what, "ms": round(ms, 4), "floor_ms": round(floor, 4)})
        print("%-52s %9.3f ms   byte floor %8.3f ms (%5.1f%%)" % (what, ms, floor, 100 * floor / ms), flush=True)

    ws = torch.empty(L.evk_cmax_workspace_bytes(180, 240), dtype=torch.uint8, device=dev)
    res = torch.empty(16 * 32, dtype=torch.float64, device=dev)
    rot = (ctypes.c_double * 3)(130.0, 85.0, 5.0)
    xyz = (ctypes.c_double * 6)(20.0, -10.0, 4.0, 3.0, 120.0, 90.0)
    models = {"rotation": (_lib.WARP_ROTATION, rot, 3), "xyztheta": (_lib.WARP_XYZTHETA, xyz, 6)}
    for N in [int(v) for v in a.sizes.split(",")]:
        g = torch.Generator(device=dev).manual_seed(7)
        t64 = torch.sort(torch.rand(N, device=dev, generator=g, dtype=torch.float64)).values * 0.05
        x64 = torch.rand(N, device=dev, generator=g, dtype=torch.float64) * 239
        y64 = torch.rand(N, device=dev, generator=g, dtype=torch.float64) * 179
        p64 = (torch.randint(0, 2, (N,), device=dev, generator=g) * 2 - 1).double()
        tl = float(t64[-1])
        x32, y32, p32, t32 = x64.float(), y64.float(), p64.float(), (t64 - tl).float()
        ev64 = [v.data_ptr() for v in (x64, y64, t64, p64)]
        ev32 = [v.data_ptr() for v in (x32, y32, t32, p32)]
        tag = "%dM" % (N // 1000000) if N >= 1000000 else str(N)
        for prec, ev, bpe in (("f64", ev64, 32), ("f32", ev32, 16)):
            for lib_name, lib in (("", L),) + ((("parent ", base),) if base is not None else ()):
                for fl, nm, passes in ((0, "f", 1), (_lib.CMAX_WANT_GRAD, "f+g", 1)):
                    if prec == "f64":
                        def run(lib=lib, fl=fl):
                            _lib.check(lib.evk_cmax_linvel_variance_f64(*ev, N, 1.0, 60.0, -35.0, tl, 180, 240, 180, 240, 1.0, fl,
                                                                        res.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None))
                    else:
                        def run(lib=lib, fl=fl):
                            _lib.check(lib.evk_cmax_linvel_variance_f32(*ev, N, 1.0, 60.0, -35.0, 180, 240, 180, 240, 1.0, fl,
                                                                        res.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None))
                    report("%s %s %slinvel %s" % (tag, prec, lib_name, nm), timeit(run), passes * N * bpe)
            if base is not None:
                # the same two builds once more, in the other order
                for lib_name, lib in (("parent ", base), ("", L)):
                    for fl, nm in ((0, "f"), (_lib.CMAX_WANT_GRAD, "f+g")):
                        if prec == "f64":
                            def run(lib=lib, fl=fl):
                                _lib.check(lib.evk_cmax_linvel_variance_f64(*ev, N, 1.0, 60.0, -35.0, tl, 180, 240, 180, 240, 1.0, fl,
                                                                            res.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None))
                        else:
                            def run(lib=lib, fl=fl):
                                _lib.check(lib.evk_cmax_linvel_variance_f32(*ev, N, 1.0, 60.0, -35.0, 180, 240, 180, 240, 1.0, fl,
                                                                            res.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None))
                        report("%s %s %slinvel %s (again)" % (tag, prec, lib_name, nm), timeit(run), N * bpe)
            for mname, (code, model, nd) in models.items():
                def run(fl, code=code, model=model):
                    if prec == "f64":
                        _lib.check(L.evk_cmax_warp_objective_f64(*ev, N, 1.0, code, ctypes.addressof(model), tl, 180, 240, 180, 240, 1.0, fl,
                                                                 0, 0.0, res.data_ptr(), None, ws.data_ptr(), ws.numel(), None))
                    else:
                        _lib.check(L.evk_cmax_warp_objective_f32(*ev, N, 1.0, code, ctypes.addressof(model), 180, 240, 180, 240, 1.0, fl,
                                                                 0, 0.0, res.data_ptr(), None, ws.data_ptr(), ws.numel(), None))
                report("%s %s %s f" % (tag, prec, mname), timeit(lambda: run(0)), N * bpe)
                report("%s %s %s f+g" % (tag, prec, mname), timeit(lambda: run(_lib.CMAX_WANT_GRAD)), 2 * N * bpe)
                report("%s %s %s gradient pass alone" % (tag, prec, mname),
                       kernel_ms(lambda: run(_lib.CMAX_WANT_GRAD), "cmax_grad_pass_kernel"), N * bpe)
                if prec == "f64":
                    batch = (ctypes.c_double * (32 * nd))(*(list(model) * 32))

                    def runb(code=code, batch=batch):
                        _lib.check(L.evk_cmax_warp_objective_batch_f64(*ev, N, 1.0, code, ctypes.addressof(batch), 32, tl, 180, 240, 180,
                                                                       240, 1.0, 0, 0, 0.0, res.data_ptr(), ws.data_ptr(), ws.numel(), None))
                    report("%s %s %s batch of 32 models (f)" % (tag, prec, mname), timeit(runb, iters=3, warm=1), N * bpe)
        del x64, y64, t64, p64, x32, y32, p32, t32
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_cmax_warps.json"), "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
