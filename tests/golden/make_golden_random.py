"""Generate the reference outputs behind the randomised oracle tests by running the UNMODIFIED reference
(TimoStoff/event_utils, loaded through oracle/ref_loader.py):

    EVK_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_random.py

  reference_random.npz  tests/test_oracle_vs_reference.py
  edge_cases.npz        tests/test_edge_cases_cpu.py
  reference_lines.json  tests/test_citations.py (line count of every .py file of the reference)

The tests regenerate the inputs from their seeds (conftest.make_events, edge_cases.cases); only the reference's
outputs are stored.  An output of more than SAMPLE cells is stored at a fixed, seeded sample of its cells (flat
indices beside the values), which keeps every file well under 1 MB.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from conftest import make_events  # noqa: E402
from edge_cases import cases as edge_cases  # noqa: E402
from oracle import ref_loader  # noqa: E402

SAMPLE = 4096
ref = ref_loader.load()
torch.set_num_threads(1)


def sample_idx(size, seed):
    if size <= SAMPLE:
        return np.arange(size, dtype=np.int32)
    return np.sort(np.random.default_rng(seed).choice(size, SAMPLE, replace=False)).astype(np.int32)


def put(out, key, arr, seed):
    arr = np.asarray(arr)
    idx = sample_idx(arr.size, seed)
    out[key + "_idx"] = idx
    out[key + "_shape"] = np.array(arr.shape, dtype=np.int64)
    out[key] = arr.ravel()[idx]


def save(name, **kw):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **kw)
    print("%-28s %8.1f KB" % (name, os.path.getsize(path) / 1024))


# ---- tests/test_oracle_vs_reference.py -----------------------------------------------------------
out = {}
for seed, n, B, H, W in [(1, 200000, 5, 260, 346), (2, 50000, 7, 180, 240), (3, 1000, 2, 10, 12)]:
    x, y, t, p = make_events(seed, n, H, W)
    v = ref.voxel_grid.events_to_voxel_torch(*(torch.from_numpy(a) for a in (x, y, t, p)), B, sensor_size=(H, W)).numpy()
    put(out, "voxel_torch_%d" % seed, v, seed)

rng = np.random.default_rng(1234)
n = 100000
xs, ys = rng.integers(0, 346, n), rng.integers(0, 260, n)
ts = np.sort(rng.random(n))
ps = rng.integers(0, 2, n) * 2 - 1.0
put(out, "voxel_numpy", ref.voxel_grid.events_to_voxel(xs, ys, ts, ps, 5, sensor_size=(260, 346)), 4)

IMAGE_KW = [dict(), dict(interpolation='bilinear'), dict(padding=False), dict(interpolation='bilinear', padding=False),
            dict(clip_out_of_range=False)]
for k, kw in enumerate(IMAGE_KW):
    x, y, t, p = make_events(5, 100000, 180, 240, pol="real")
    if kw.get("clip_out_of_range", True):
        x[::7] += 4
    a = ref.image.events_to_image_torch(torch.from_numpy(x), torch.from_numpy(y), torch.from_numpy(p), **kw).numpy()
    put(out, "image_%d" % k, a, 10 + k)

x, y, t, p = make_events(6, 50000, 180, 240)
flow = torch.from_numpy((np.random.default_rng(6).standard_normal((2, 180, 240)) * 30).astype(np.float32))
xw, yw = ref.optic_flow.warp_events_flow_torch(*(torch.from_numpy(a) for a in (x, y, t, p)), flow)
put(out, "flow_x", xw.numpy(), 20)
put(out, "flow_y", yw.numpy(), 21)

rows = []                       # sigma, vx, vy, f, g0, g1, gradient scale
x, y, t, p = make_events(7, 100000, 180, 240, dtype=np.float64)
obj, warp = ref.objectives.variance_objective(), ref.warps.linvel_warp()
for sigma in (1.0, 0.0, 3.0):
    for params in [(30.0, -20.0), (-400.0, 900.0)]:
        f = obj.evaluate_function(params, x, y, t, p, warp, (180, 240), sigma)
        g = obj.evaluate_gradient(params, x, y, t, p, warp, (180, 240), sigma)
        iwe, d = ref.objectives.get_iwe(params, x, y, t, p, warp, (180, 240), compute_gradient=True)
        scale = np.sqrt(np.mean((2 * (iwe - iwe.mean())) ** 2) * np.mean(d ** 2))
        rows.append([sigma, params[0], params[1], f, g[0], g[1], scale])
out["cmax"] = np.array(rows)

import importlib  # noqa: E402
ref_cmax = importlib.import_module("lib.contrast_max.events_cmax")
rng = np.random.default_rng(0)
ranges = []
for _ in range(500):
    axis = np.sort(rng.uniform(-200, 200, rng.integers(3, 9)))
    value = rng.choice(axis) if rng.random() < 0.7 else rng.uniform(-250, 250)
    ranges.append(np.asarray(ref_cmax.find_new_range(axis, value), dtype=np.float64))
out["find_new_range"] = np.array(ranges)

bd = importlib.import_module("lib.data_loaders.base_dataset")
rng = np.random.default_rng(3)
ts = np.sort(rng.uniform(5.0, 7.5, 20000))
ts[100:110] = ts[100]


class Probe(bd.BaseVoxelDataset):                       # the table code only, no recording behind it
    def __init__(self):
        self.num_events, self.t0, self.tk = len(ts), ts[0], ts[-1]
        self.duration = self.tk - self.t0
        self.has_frames = False

    def find_ts_index(self, timestamp):
        return np.searchsorted(ts, timestamp)


d = Probe()
for k, w in ((1000, 0), (1500, 500), (333, 33)):
    d.set_voxel_method({"method": "k_events", "k": k, "sliding_window_w": w})
    out["windows_k_%d_%d" % (k, w)] = np.asarray(d.event_indices, dtype=np.int64)
for t_, w in ((0.1, 0.0), (0.25, 0.05), (0.013, 0.0)):
    d.set_voxel_method({"method": "t_seconds", "t": t_, "sliding_window_t": w})
    out["windows_t_%g_%g" % (t_, w)] = np.asarray(d.event_indices, dtype=np.int64)
for nf in (1, 7, 40):
    d.set_voxel_method({"method": "fixed_frames", "num_frames": nf})
    out["windows_f_%d" % nf] = np.asarray(d.event_indices, dtype=np.int64)
d.frame_ts = np.concatenate((np.sort(rng.uniform(5.0, 7.5, 30)), [9.0]))
d.num_frames = len(d.frame_ts)
d.set_voxel_method({"method": "between_frames"})
out["windows_frame_ts"] = d.frame_ts
out["windows_between"] = np.asarray(d.event_indices, dtype=np.int64)

rows = []                       # objective index, vx, vy, sigma (nan = None), f, g0, g1 (nan = not compared)
NAMES = ["rms", "sos", "soe", "moa", "isoa", "sosa", "r1"]
x, y, t, p = make_events(17, 60000, 180, 240, dtype=np.float64)
for i, name in enumerate(NAMES):
    obj, warp = getattr(ref.objectives, name + "_objective")(), ref.warps.linvel_warp()
    for params in [(25.0, -40.0), (-300.0, 120.0)]:
        for sigma in (None, 0.0, 1.7):
            f = obj.evaluate_function(params, x, y, t, p, warp, (180, 240), sigma)
            g = [np.nan, np.nan]
            if name in ("rms", "soe", "isoa", "sosa"):
                g = obj.evaluate_gradient(params, x, y, t, p, warp, (180, 240), sigma)
            rows.append([i, params[0], params[1], np.nan if sigma is None else sigma, f, g[0], g[1]])
out["objectives"] = np.array(rows)
save("reference_random", **out)


# ---- tests/test_edge_cases_cpu.py: results (flat, per case and output) or the error raised ----------------------------
def run(fn):
    try:
        return np.asarray(fn(), dtype=np.float32).ravel(), 0
    except (IndexError, ValueError, RuntimeError):
        return np.zeros(0, np.float32), 1


vals, raised, lens = [], [], []
for c in edge_cases(2024, 300):
    T = [torch.from_numpy(c[k]) for k in "xytp"]
    hw = (c["H"], c["W"])
    outs = [run(lambda: ref.voxel_grid.events_to_voxel_torch(*T, c["B"], sensor_size=hw).numpy())]
    for interp in (None, "bilinear"):
        kw = dict(sensor_size=hw, clip_out_of_range=c["clip"], interpolation=interp, padding=c["padding"])
        outs.append(run(lambda: ref.image.events_to_image_torch(T[0], T[1], T[3], **kw).numpy()))
    for v, e in outs:
        vals.append(v)
        raised.append(e)
        lens.append(v.size)
save("edge_cases", values=np.concatenate(vals), raised=np.array(raised, np.uint8), lengths=np.array(lens, np.int32))

# ---- tests/test_citations.py: line count of every .py file of the reference --------------------------------------------
lines = {}
for dp, _, files in os.walk(ref_loader.REF_ROOT):
    for f in files:
        if f.endswith(".py"):
            path = os.path.join(dp, f)
            lines[os.path.relpath(path, ref_loader.REF_ROOT)] = sum(1 for _ in open(path, errors="replace"))
with open(os.path.join(HERE, "reference_lines.json"), "w") as f:
    json.dump(dict(sorted(lines.items())), f, indent=0)
    f.write("\n")
print("reference_lines.json         %d files" % len(lines))
