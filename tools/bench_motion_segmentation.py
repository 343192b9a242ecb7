"""Motion segmentation entries (evk_cmax_motion_segment_*) and the EM fit (motion_segmentation_fit_torch) against what a
user writes without them: M calls of the single-model entries on p * w[:, m].

    python tools/bench_motion_segmentation.py [--reps 20] [--out DIR]

Rows (DESIGN.md section 6), rotation model, uniform events over the sensor, random memberships:
    64 windows x 100 k events, 180x240, M = 2 and M = 4
    16 windows x 500 k events, 480x640, M = 4
Per entry: the median of --reps CUDA-event timings of one call (forward; gradient with and without the membership
gradient; a 32-wide candidates pass, i.e. 32 // M candidates per model; the assignment), beside the time the events'
bytes take at the data sheet's 3.35 TB/s (16 + 4M bytes per event for the passes that read each event once).  The
comparison arm runs in the same process, alternated with the new entries: M forward + gradient calls of
evk_cmax_motion_objective_f32 / _grad_f32, and M candidates calls of evk_cmax_motion_candidates_f32 of the same total
width, each on p * w[:, m] formed by torch as a user would.  One EM round (em_iters = 1) and the whole fit
(em_iters = 10, max_iter = 20) are wall times that end in a device synchronise.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200 import _lib  # noqa: E402
from event_utils_b200.contrast_max import motion_segmentation_fit_torch, pure_rotation_warp  # noqa: E402

ROWS = [dict(B=64, per=100_000, H=180, W=240, M=2), dict(B=64, per=100_000, H=180, W=240, M=4),
        dict(B=16, per=500_000, H=480, W=640, M=4)]
HBM = 3.35e12


def events(B, per, H, W, seed):
    rng = np.random.default_rng(seed)
    n = B * per
    x = torch.from_numpy((rng.random(n) * (W - 1)).astype(np.float32)).cuda()
    y = torch.from_numpy((rng.random(n) * (H - 1)).astype(np.float32)).cuda()
    d = torch.from_numpy((-rng.random(n) * 0.05).astype(np.float32)).cuda()
    p = torch.ones(n, device="cuda")
    off = torch.arange(0, n + 1, per, dtype=torch.int64, device="cuda")
    return x, y, d, p, off


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run_row(row, reps):
    L = _lib.lib()
    B, per, H, W, M = row["B"], row["per"], row["H"], row["W"], row["M"]
    n = B * per
    K = 3
    x, y, d, p, off = events(B, per, H, W, 7)
    rng = np.random.default_rng(8)
    w = torch.from_numpy(rng.random((n, M)).astype(np.float32)).cuda()
    w /= w.sum(1, keepdim=True)
    params = torch.tensor([[[W / 2 + 10 * m, H / 2 - 5 * m, 2.0 + m] for m in range(M)]] * B, dtype=torch.float64, device="cuda")
    J = 32 // M
    cand = (params.unsqueeze(2) * torch.linspace(0.9, 1.1, J, dtype=torch.float64, device="cuda").view(1, 1, J, 1)).contiguous()
    f = torch.empty((B, M), dtype=torch.float64, device="cuda")
    fc = torch.empty((B, M, J), dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, M, H + 1, W + 1), device="cuda")
    gf = torch.ones((B, M), device="cuda")
    gp = torch.empty((B, M, K), dtype=torch.float64, device="cuda")
    gw = torch.zeros((n, M), device="cuda")
    wout = torch.empty((n, M), device="cuda")
    ws = torch.empty(L.evk_cmax_motion_segment_workspace_bytes(B, M, H, W), dtype=torch.uint8, device="cuda")
    wsc = torch.empty(L.evk_cmax_motion_segment_candidates_workspace_bytes(B, M, J, H, W), dtype=torch.uint8, device="cuda")
    P = _lib.ptr
    st = _lib.stream()
    ev = (P(x), P(y), P(d), P(p), P(w), M, P(off), B, n, _lib.WARP_ROTATION)
    tail = (K, 0.0, 0.0, H, W, 1.0, _lib.OBJ_VARIANCE, 0.0)
    new = {
        "forward": lambda: _lib.check(L.evk_cmax_motion_segment_f32(*ev, P(params), *tail, P(f), P(iwe), P(ws), ws.numel(), st)),
        "grad": lambda: _lib.check(L.evk_cmax_motion_segment_grad_f32(*ev, P(params), *tail, P(iwe), P(gf), P(gp), None, P(ws),
                                                                      ws.numel(), st)),
        "grad_weights": lambda: _lib.check(L.evk_cmax_motion_segment_grad_f32(*ev, P(params), *tail, P(iwe), P(gf), P(gp), P(gw),
                                                                              P(ws), ws.numel(), st)),
        "candidates_32": lambda: _lib.check(L.evk_cmax_motion_segment_candidates_f32(*ev, P(cand), J, *tail, P(fc), P(wsc), wsc.numel(),
                                                                                     st)),
        "assign": lambda: _lib.check(L.evk_cmax_motion_segment_assign_f32(P(x), P(y), P(d), M, P(off), B, n, _lib.WARP_ROTATION,
                                                                          P(params), K, 0.0, 0.0, H, W, P(iwe), 1.0, 1e-6, P(wout),
                                                                          P(ws), ws.numel(), st)),
    }
    new["forward"]()
    # the comparison arm: M single-model calls on p * w[:, m]
    prm_m = [params[:, m].contiguous() for m in range(M)]
    cand_m = [cand[:, m].contiguous() for m in range(M)]
    f1 = torch.empty(B, dtype=torch.float64, device="cuda")
    f1c = torch.empty((B, J), dtype=torch.float64, device="cuda")
    iwe1 = torch.empty((B, H + 1, W + 1), device="cuda")
    g1 = torch.ones(B, device="cuda")
    gp1 = torch.empty((B, K), dtype=torch.float64, device="cuda")
    ws1 = torch.empty(L.evk_cmax_motion_objective_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    ws1c = torch.empty(L.evk_cmax_motion_candidates_workspace_bytes(B, J, H, W), dtype=torch.uint8, device="cuda")

    def per_model_fg():
        for m in range(M):
            pm = (p * w[:, m]).contiguous()
            e1 = (P(x), P(y), P(d), P(pm), P(off), B, n, _lib.WARP_ROTATION, P(prm_m[m])) + tail
            _lib.check(L.evk_cmax_motion_objective_f32(*e1, P(f1), P(iwe1), P(ws1), ws1.numel(), st))
            _lib.check(L.evk_cmax_motion_objective_grad_f32(*e1, P(iwe1), P(g1), P(gp1), P(ws1), ws1.numel(), st))

    def per_model_cand():
        for m in range(M):
            pm = (p * w[:, m]).contiguous()
            _lib.check(L.evk_cmax_motion_candidates_f32(P(x), P(y), P(d), P(pm), P(off), B, n, _lib.WARP_ROTATION, P(cand_m[m]), J,
                                                        *tail, P(f1c), P(ws1c), ws1c.numel(), st))
    # the same values: the new forward against the arm's per model
    for m in range(M):
        pm = (p * w[:, m]).contiguous()
        _lib.check(L.evk_cmax_motion_objective_f32(P(x), P(y), P(d), P(pm), P(off), B, n, _lib.WARP_ROTATION, P(prm_m[m]), *tail,
                                                   P(f1), P(iwe1), P(ws1), ws1.numel(), st))
        assert torch.allclose(f1, f[:, m], rtol=1e-6, atol=0), m
    times = {k: [] for k in list(new) + ["fg_new", "fg_per_model", "cand_per_model"]}
    fg_new = lambda: (new["forward"](), new["grad"]())
    for _ in range(3):                                      # alternate the two arms
        for k, fn in new.items():
            times[k].append(median_ms(fn, reps))
        times["fg_new"].append(median_ms(fg_new, reps))
        times["fg_per_model"].append(median_ms(per_model_fg, reps))
        times["cand_per_model"].append(median_ms(per_model_cand, reps))
    out = {k: float(np.median(v)) for k, v in times.items()}
    floor_one_read = n * (16 + 4 * M) / HBM * 1e3
    out["floor_ms_16_plus_4M"] = floor_one_read
    out["floor_ms_assign_reads_12_writes_4M"] = n * (12 + 4 * M) / HBM * 1e3
    # EM: one round and the whole fit, wall time ending in a synchronise
    warp = pure_rotation_warp()
    x0 = params[0]
    kw = dict(batch_end_indices=off[1:], img_size=(H, W), param_scale=[0.5, 0.5, 0.05])

    def fit(em):
        torch.cuda.synchronize()
        t = time.perf_counter()
        motion_segmentation_fit_torch(x, y, d, p, warp, x0, em_iters=em, max_iter=20, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3
    fit(1)
    out["em_round_ms"] = float(np.median([fit(1) for _ in range(3)]))
    out["fit_10_rounds_ms"] = fit(10)
    return dict(row, events=n, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card: %s" % card)
    rows = []
    for row in ROWS:
        r = run_row(row, a.reps)
        r["card"] = card
        print(json.dumps(r))
        rows.append(r)
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_motion_segmentation.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
