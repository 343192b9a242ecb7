"""Where does the time of one objective evaluation through the python API go? (development tool)"""
import os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from event_utils_b200 import _lib
from event_utils_b200.contrast_max import objectives as O
from event_utils_b200.contrast_max.warps import linvel_warp

rng = np.random.default_rng(0)
for n in (15_000, 1_000_000):
    xs, ys = rng.random(n) * 239, rng.random(n) * 179
    ts, ps = np.sort(rng.random(n)) * 0.1, rng.integers(0, 2, n) * 2.0 - 1
    obj, warp = O.variance_objective(), linvel_warp()
    args = (xs, ys, ts, ps, warp, (180, 240), 1.0)
    obj.evaluate_function((1.0, 1.0), *args)
    K = 300
    t0 = time.perf_counter()
    for i in range(K):
        obj.evaluate_function((40 + 0.01 * i, -20.0), *args)
    tot = (time.perf_counter() - t0) / K
    # pieces
    t0 = time.perf_counter()
    for i in range(K):
        O._device_events(xs, ys, ts, ps)
    fp = (time.perf_counter() - t0) / K
    L = _lib.lib()
    ev = O._device_events(xs, ys, ts, ps)
    ws = _lib.scratch("cmax_ws", L.evk_cmax_workspace_bytes(180, 240), ev.x.device)
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(K):
        _lib.check(L.evk_cmax_linvel_objective_f64(ev.x.data_ptr(), ev.y.data_ptr(), ev.t.data_ptr(), ev.p.data_ptr(), n, 1.0, 40.0 + 0.01 * i, -20.0,
                                                   ev.t_last, 180, 240, 180, 240, 1.0, _lib.CMAX_WANT_GRAD, 0, 0.0, res.data_ptr(), None, None,
                                                   ws.data_ptr(), ws.numel(), None))
    launch = (time.perf_counter() - t0) / K
    torch.cuda.synchronize()
    gpu_total = (time.perf_counter() - t0) / K
    t0 = time.perf_counter()
    for i in range(K):
        _lib.check(L.evk_cmax_linvel_objective_f64(ev.x.data_ptr(), ev.y.data_ptr(), ev.t.data_ptr(), ev.p.data_ptr(), n, 1.0, 40.0 + 0.01 * i, -20.0,
                                                   ev.t_last, 180, 240, 180, 240, 1.0, _lib.CMAX_WANT_GRAD, 0, 0.0, res.data_ptr(), None, None,
                                                   ws.data_ptr(), ws.numel(), None))
        r = res.cpu().numpy()
    sync_each = (time.perf_counter() - t0) / K
    print("n=%8d  api %.1f us/eval | fingerprint+cache %.1f us | C call (async, back to back) %.1f us, GPU-bound %.1f us | C call + D2H sync each %.1f us"
          % (n, tot * 1e6, fp * 1e6, launch * 1e6, gpu_total * 1e6, sync_each * 1e6))

# grid search: 25 candidates in one pass vs 25 separate evaluations
from event_utils_b200.contrast_max.events_cmax import grid_search_initial
for n in (15_000, 1_000_000):
    xs, ys = rng.random(n) * 239, rng.random(n) * 179
    ts, ps = np.sort(rng.random(n)) * 0.1, rng.integers(0, 2, n) * 2.0 - 1
    obj, warp = O.variance_objective(), linvel_warp()
    grid_search_initial(xs, ys, ts, ps, warp, obj, (180, 240))
    t0 = time.perf_counter()
    for _ in range(20):
        out = grid_search_initial(xs, ys, ts, ps, warp, obj, (180, 240))
    tb = (time.perf_counter() - t0) / 20
    t0 = time.perf_counter()
    for _ in range(20):
        ev = [obj.evaluate_function(p, xs, ys, ts, ps, warp, (180, 240), 1.0) for p in out["params"]]
    tl = (time.perf_counter() - t0) / 20
    print("n=%8d  grid_search_initial (25 points): batched %.0f us, one evaluation per point %.0f us" % (n, tb * 1e6, tl * 1e6))
