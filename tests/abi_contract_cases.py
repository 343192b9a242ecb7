"""The case table of the ABI contract tests (tests/test_abi_contract_cpu.py, tests/test_gpu_abi_contract.py).

include/evk.h promises, besides the numbers, where every device entry writes, what it reads and which stream it uses:
outputs are fully overwritten unless EVK_ACCUMULATE is set, the workspace is the query's size and 256-byte aligned, the
query returns 0 for the arguments its entries reject, every argument is checked before any CUDA call, and all work goes
on the caller's stream without a synchronisation.  For every device entry this module has either builders of calls at
the shapes where the workspace carving changes, or an entry in EXCLUDED with the reason it is never run this way.

A call is described by name: `values` maps the parameter names of the entry's prototype in include/evk.h to numpy
arrays (uploaded to the device as they are), Python scalars, or `Out` records of the outputs the entry writes.  The
harness adds workspace, workspace_bytes and stream.  The workspace query takes its arguments from the same names.

The batched losses are the entries whose workspace is carved by batch_obj_carve (evk_cmax.cu) into up to nine aliased
regions; their limits (limit_points) are swept by the CPU test at the limit and one past it.
"""
import os
import re

import numpy as np

from candidate_checks import draw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OVERWRITE, ACCUMULATE, SCRATCH = "overwrite", "accumulate", "scratch"    # SCRATCH: caller scratch, never compared

# entries without a case, each with its reason (a new entry that is neither here nor in the table fails the coverage test)
EXCLUDED = {
    "evk_version": "no device work",
    "evk_last_error": "no device work",
    "evk_device_check": "queries the device, writes no buffer and enqueues nothing",
    "evk_prof_enable": "measurement hook: toggles host-side counters",
    "evk_prof_collect": "measurement hook: synchronises its own events by design (bench.py only)",
    "evk_peer_barrier": "a cross-GPU spin-wait protocol: poisoned slots could stall it until the watchdog fires",
    "evk_voxel_fold_allreduce_f32": "the peer / multicast fold: reads other ranks' workspaces and must follow a cross-GPU "
                                    "barrier, a spin-wait protocol",
    # (evk_cmax_peer_tail_f32 reads its ranks' images through a host table of device pointers; at world = 1 it needs no
    # barrier, and it has cases below)
    "evk_pipeline_create": "host pipeline: synchronous by design (allocates its staging buffers)",
    "evk_pipeline_destroy": "host pipeline: synchronous by design",
    "evk_voxel_host_f32": "host pipeline: synchronous by design, writes host memory",
    "evk_voxel_host_packed_f32": "host pipeline: synchronous by design, writes host memory",
    "evk_host_upload": "host pipeline: synchronous by design",
    "evk_host_hash64": "host only, no device work",
    "evk_host_hash64_multi": "host only, no device work",
    "evk_host_copy": "host only, no device work",
}


class Out:
    """an output of `nbytes` bytes, read back as `dtype`; mode OVERWRITE or ACCUMULATE"""

    def __init__(self, nbytes, dtype, mode=OVERWRITE):
        self.nbytes, self.dtype, self.mode = int(nbytes), np.dtype(dtype), mode


class Host:
    """an array the entry reads from HOST memory (parameter tables of the single-window contrast entries)"""

    def __init__(self, arr):
        self.arr = np.ascontiguousarray(arr)


class DevicePointers:
    """a HOST table of the device addresses of the named inputs (the peer tables of evk_cmax_peer_tail_f32)"""

    def __init__(self, *names):
        self.names = names


class Case:
    """One call of `entry`.  rtol: 0 for entries whose outputs repeat bit for bit, else the f32-atomics tolerance of
    the family, relative to the largest magnitude of each output."""

    def __init__(self, entry, tag, values, rtol=0.0):
        # a builder may share one dict of values between entries: outputs the entry does not take are dropped
        names = set(protos()[entry])
        values = {k: v for k, v in values.items() if not isinstance(v, Out) or k in names}
        self.entry, self.tag, self.values, self.rtol = entry, tag, values, rtol

    @property
    def id(self):
        return "%s[%s]" % (self.entry, self.tag)

    def outputs(self):
        return {k: v for k, v in self.values.items() if isinstance(v, Out)}

    def compared(self):
        return {k: v for k, v in self.outputs().items() if v.mode != SCRATCH}

    def query(self):
        return workspace_query(self.entry)

    def workspace_bytes(self, L):
        """the workspace the entry's query asks for at this call (0 without a query)"""
        q = self.query()
        return int(getattr(L, q)(*query_args(q, self.values))) * WORKSPACE_FACTOR.get(self.entry, 1) if q else 0


def prototypes():
    """entry -> list of parameter names, from include/evk.h"""
    src = open(os.path.join(ROOT, "include", "evk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|size_t|uint64_t|const char \*|void)\s*\*?\s*(evk_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src,
                         flags=re.S):
        params = [p.strip() for p in m.group(2).replace("\n", " ").split(",")]
        out[m.group(1)] = [] if params in ([""], ["void"]) else [re.findall(r"[A-Za-z_][A-Za-z0-9_]*", p)[-1] for p in params]
    return out


_PROTOS = None


def protos():
    global _PROTOS
    if _PROTOS is None:
        _PROTOS = prototypes()
    return _PROTOS


def workspace_query(entry):
    """the query that sizes `entry`'s workspace, or None when the entry takes no workspace"""
    P = protos()
    if entry in QUERY_OF:
        return QUERY_OF[entry]
    if "workspace" not in P[entry]:
        return None
    stem = entry[:-4] if entry.endswith(("_f32", "_f64")) else entry
    for s in (stem, re.sub(r"_(grad|assign)$", "", stem), re.sub(r"_(grad|counts)$", "", stem)):
        if s + "_workspace_bytes" in P:
            return s + "_workspace_bytes"
    raise KeyError("no workspace query for %s" % entry)


def query_args(query, values):
    return [values[n] for n in protos()[query]]


# ---- the batched losses ---------------------------------------------------------------------------------------------
# family -> its entries.  Every entry of a family takes its arguments from one scene.
BATCHED = {
    "flow": ["evk_cmax_flow_objective_f32", "evk_cmax_flow_objective_grad_f32"],
    "flow_ts": ["evk_flow_timestamp_objective_f32", "evk_flow_timestamp_objective_grad_f32"],
    "motion": ["evk_cmax_motion_objective_f32", "evk_cmax_motion_objective_grad_f32", "evk_cmax_motion_candidates_f32"],
    "motion_depth": ["evk_cmax_motion_depth_objective_f32", "evk_cmax_motion_depth_objective_grad_f32",
                     "evk_cmax_motion_depth_candidates_f32"],
    "motion_ts": ["evk_motion_timestamp_objective_f32", "evk_motion_timestamp_objective_grad_f32",
                  "evk_motion_timestamp_candidates_f32"],
    "motion_ts_depth": ["evk_motion_timestamp_depth_objective_f32", "evk_motion_timestamp_depth_objective_grad_f32",
                        "evk_motion_timestamp_depth_candidates_f32"],
    "segment": ["evk_cmax_motion_segment_f32", "evk_cmax_motion_segment_grad_f32", "evk_cmax_motion_segment_candidates_f32",
                "evk_cmax_motion_segment_assign_f32"],
    "grid_flow": ["evk_cmax_grid_flow_objective_f32", "evk_cmax_grid_flow_objective_grad_f32",
                  "evk_cmax_grid_flow_candidates_f32"],
    "grid_flow_ts": ["evk_grid_flow_timestamp_objective_f32", "evk_grid_flow_timestamp_objective_grad_f32",
                     "evk_grid_flow_timestamp_candidates_f32"],
    "depth_grid": ["evk_cmax_depth_grid_objective_f32", "evk_cmax_depth_grid_objective_grad_f32",
                   "evk_cmax_depth_grid_candidates_f32", "evk_cmax_depth_grid_joint_grad_f32",
                   "evk_cmax_depth_grid_joint_candidates_f32"],
    "depth_grid_ts": ["evk_depth_grid_timestamp_objective_f32", "evk_depth_grid_timestamp_objective_grad_f32",
                      "evk_depth_grid_timestamp_candidates_f32"],
}
TIMESTAMP = {"flow_ts", "motion_ts", "motion_ts_depth", "grid_flow_ts", "depth_grid_ts"}
GRID = {"grid_flow", "grid_flow_ts", "depth_grid", "depth_grid_ts"}
MAX_GRID_NODES = 4096          # gh gw of the grid losses
MAX_GRID_CAND_NODES = 12288    # n_cand gh gw of the grid candidates passes
MAX_CANDIDATES = 32
MAX_MODELS = 8


def family_of(entry):
    for fam, entries in BATCHED.items():
        if entry in entries:
            return fam
    return None


def kind_of(entry):
    if "candidates" in entry:
        return "cand"
    if "assign" in entry:
        return "assign"
    return "grad" if "grad" in entry else "fwd"


def image_cap(fam):
    """the largest batch (times candidates, times models) of the family's tail images"""
    return 32767 if fam in TIMESTAMP else 65535


# Shapes where the carving changes: a 2x2 sensor, an odd canvas and the full 180x240 one; a single window and skewed
# windows (an empty and a one-event window beside larger ones); J = 1 and 32 candidates and n_cand gh gw at its limit;
# 2x2 node grids and grids as fine as the sensor; 2 and 8 segmentation models.
SHAPES = [
    # tag, H, W, window sizes, J, (gh, gw), M
    ("2x2-b1-J32-M8", 2, 2, [7], 32, (2, 2), 8),
    ("37x53-skew-J1-M2", 37, 53, [40, 0, 1, 25], 1, (2, 2), 2),
    ("37x53-skew-J32-fullgrid", 37, 53, [40, 0, 1, 25], 32, (37, 53), 1),     # the grid families: J = 6
    ("180x240-b2-Jmaxnodes", 180, 240, [3000, 1], 3, (64, 64), 2),
]


def _scene(fam, H, W, sizes, J, grid, M, seed):
    rng = np.random.default_rng(seed)
    sizes = np.asarray(sizes, np.int64)
    n = int(sizes.sum())
    x, y, d, p, rho = draw(rng, n, H, W)
    B = len(sizes)
    f32, f64 = np.float32, np.float64
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    gh, gw = grid
    v = dict(x=x, y=y, t_rel=d, p=p, offsets=off, batch=B, n_events=n, H=H, W=W, sigma=1.0, blur_sigma=1.0,
             objective=0, obj_param=1.0, cx=(W - 1) / 2.0, cy=(H - 1) / 2.0)
    Hc, Wc = H + 1, W + 1
    if fam in TIMESTAMP:
        v["tau"] = rng.random(n).astype(f32)
        v["ts_img"] = rng.random((B, 2, Hc, Wc)).astype(f32)
        v["cnt_img"] = (1 + rng.random((B, 2, Hc, Wc))).astype(f32)
    else:
        v["iwe"] = rng.random((B, M if fam == "segment" else 1, Hc, Wc)).astype(f32)
    v["grad_f"] = rng.uniform(-1, 1, B * (M if fam == "segment" else 1)).astype(f32)
    if fam in ("flow", "flow_ts"):
        v["flow"] = rng.uniform(-3, 3, (B, 2, H, W)).astype(f32)
    elif fam in ("motion", "motion_ts", "segment"):
        v["warp"], v["K"] = 4, 6           # EVK_WARP_AFFINE
        shape = (B, M) if fam == "segment" else (B,)
        rows = np.concatenate([rng.uniform(-5, 5, shape + (2,)), rng.uniform(-1, 1, shape + (4,))], axis=-1)
        v["params"] = rows
        v["cand"] = np.repeat(rows[..., None, :], J, axis=-2) + rng.uniform(-0.5, 0.5, shape + (J, 6))
    elif fam in ("motion_depth", "motion_ts_depth"):
        v["warp"], v["K"] = 7, 8           # EVK_WARP_CAMERA_MOTION
        v["inv_depth"] = rho
        rows = np.column_stack((rng.uniform(-2, 2, (B, 6)), np.full((B, 2), 0.8 * max(H, W))))
        v["params"] = rows
        v["cand"] = np.repeat(rows[:, None, :], J, axis=1)
        v["cand"][..., :6] += rng.uniform(-0.3, 0.3, (B, J, 6))
    if fam in GRID:
        v["gh"], v["gw"] = gh, gw
        if fam.startswith("grid_flow"):
            v["grid_flow"] = rng.uniform(-3, 3, (B, 2, gh, gw)).astype(f32)
            v["cand"] = rng.uniform(-3, 3, (B, J, 2, gh, gw)).astype(f32)
        else:
            v["inv_depth_grid"] = rng.uniform(0.125, 1.0, (B, gh, gw)).astype(f32)
            v["cand"] = rng.uniform(0.125, 1.0, (B, J, gh, gw)).astype(f32)
            rows = np.column_stack((rng.uniform(-2, 2, (B, 6)), np.full((B, 2), 0.8 * max(H, W))))
            v["motion"] = rows
    if fam == "segment":
        v["n_models"] = M
        v["weights"] = rng.random((n, M)).astype(f32)
        v["eps"] = 1e-3
    v["n_cand"] = J
    return v


def _outputs(entry, fam, v):
    """the Out records of `entry` in scene v"""
    B, H, W, n = v["batch"], v["H"], v["W"], v["n_events"]
    Hc, Wc = H + 1, W + 1
    M = v.get("n_models", 1)
    J = v["n_cand"]
    kind = kind_of(entry)
    o = {}
    if kind == "cand":
        o["f_out"] = Out(B * M * J * 8, np.float64)
    elif kind == "fwd":
        o["f_out"] = Out(B * M * 8, np.float64)
        if fam in TIMESTAMP:
            o["ts_out"] = Out(B * 2 * Hc * Wc * 4, np.float32)
            o["cnt_out"] = Out(B * 2 * Hc * Wc * 4, np.float32)
        else:
            o["iwe_out"] = Out(B * M * Hc * Wc * 4, np.float32)
    elif kind == "assign":
        o["weights_out"] = Out(n * M * 4, np.float32)
    else:
        if fam in ("flow", "flow_ts"):
            o["grad_flow"] = Out(B * 2 * H * W * 4, np.float32)
        elif fam.startswith("grid_flow"):
            o["grad_grid"] = Out(B * 2 * v["gh"] * v["gw"] * 4, np.float32)
        elif fam.startswith("depth_grid"):
            o["grad_grid"] = Out(B * v["gh"] * v["gw"] * 4, np.float32)
            if "joint" in entry:
                o["grad_motion"] = Out(B * 6 * 8, np.float64)
        else:
            o["grad_params"] = Out(B * M * v["K"] * 8, np.float64)
            if fam == "segment":
                o["grad_weights"] = Out(n * M * 4, np.float32)
    return o


def batched_cases(seed=0):
    """every batched entry at every SHAPE that applies to its family"""
    cases = []
    for fam, entries in BATCHED.items():
        for k, (tag, H, W, sizes, J, grid, M) in enumerate(SHAPES):
            if fam in GRID and (grid[0] > H or grid[1] > W):
                continue
            if fam in GRID:
                J = min(J, MAX_GRID_CAND_NODES // (grid[0] * grid[1]))
            if fam == "segment":
                J = max(1, min(J, MAX_CANDIDATES // M))
            else:
                M = 1
            for entry in entries:
                if "joint_candidates" in entry:
                    v = _scene(fam, H, W, sizes, J, grid, M, seed + 10 * k)
                    v["motion"] = np.repeat(v["motion"][:, None, :], J, axis=1)
                    v["motion"][..., :6] += np.random.default_rng(seed + k).uniform(-0.3, 0.3, (len(sizes), J, 6))
                else:
                    v = _scene(fam, H, W, sizes, J, grid, M, seed + 10 * k)
                v.update(_outputs(entry, fam, v))
                # f32 atomics in the event passes and f64 atomics in the gradient sums: the order of the adds varies
                cases.append(Case(entry, tag, v, rtol=2e-5))
    return cases


# ---- limits of the batched queries, for the query / refusal sweep ------------------------------------------------------

def limit_points(entry):
    """(label, overrides, accepted) of the scene at a limit of `entry` and one past it.  The base scene is accepted."""
    fam = family_of(entry)
    kind = kind_of(entry)
    cap = image_cap(fam)
    pts = []
    cand = kind == "cand"
    M = 2 if fam == "segment" else 1
    J = 4 if cand else 1
    per = M * J
    pts += [("batch=-1", dict(batch=-1), False), ("batch=0", dict(batch=0), True)]
    pts += [("batch*M*J=cap", dict(batch=cap // per), True), ("batch*M*J=cap+1", dict(batch=cap // per + 1), False)]
    if cand:
        pts += [("J=0", dict(n_cand=0), False), ("J=1", dict(n_cand=1), True)]
        jmax = MAX_CANDIDATES // M
        pts += [("J=max", dict(n_cand=jmax, batch=1), True), ("J=max+1", dict(n_cand=jmax + 1, batch=1), False)]
        # products that wrap an int: M J = 2^32 and batch J = 2^32 + 4
        pts += [("J=2^31-1", dict(n_cand=2 ** 31 - 1, batch=1), False), ("J=2^30", dict(n_cand=2 ** 30, batch=4), False)]
    if fam == "segment":
        pts += [("M=0", dict(n_models=0), False), ("M=1", dict(n_models=1), True)]
        pts += [("M=8", dict(n_models=8, n_cand=(4 if cand else 1)), True),
                ("M=9", dict(n_models=9, n_cand=1), False)]
        if cand:
            pts += [("M*J=33", dict(n_models=3, n_cand=11), False), ("M=8,J=2^29", dict(n_models=8, n_cand=2 ** 29), False)]
        else:
            pts += [("batch*M=2^32", dict(n_models=8, batch=2 ** 29), False)]
    pts += [("H=1", dict(H=1), False), ("W=1", dict(W=1), False), ("H=W=2", dict(H=2, W=2, gh=2, gw=2), True)]
    # the 2^30-pixel canvas: (H+1)(W+1) = 2^30 exactly, then one row more
    pts += [("canvas=2^30", dict(H=32767, W=32767, batch=1, n_cand=1), True),
            ("canvas>2^30", dict(H=32768, W=32767, batch=1, n_cand=1), False),
            ("canvas=40000^2", dict(H=40000, W=40000, batch=1, n_cand=1), False)]
    if fam in GRID:
        pts += [("gh=1", dict(gh=1), False), ("gw=1", dict(gw=1), False),
                ("gh=H", dict(gh=40, H=40), True), ("gh=H+1", dict(gh=41, H=40), False),
                ("gw=W", dict(gw=50, W=50), True), ("gw=W+1", dict(gw=51, W=50), False)]
        if cand:
            pts += [("J*gh*gw=max", dict(n_cand=3, gh=64, gw=64, H=64, W=64, batch=1), True),
                    ("J*gh*gw=max+", dict(n_cand=3, gh=64, gw=65, H=64, W=65, batch=1), False)]
        else:
            pts += [("gh*gw=max", dict(gh=64, gw=64, H=64, W=64), True),
                    ("gh*gw=max+", dict(gh=64, gw=65, H=64, W=65), False)]
    return pts


def sweep_values(entry, overrides):
    """the scalar arguments of `entry` at the sweep's base scene with `overrides`; pointers are left to the caller"""
    fam = family_of(entry)
    v = dict(batch=3, n_events=10, H=10, W=12, gh=3, gw=4, sigma=1.0, blur_sigma=1.0, objective=0, obj_param=1.0,
             cx=5.0, cy=4.0, n_models=2 if fam == "segment" else 1, n_cand=4 if kind_of(entry) == "cand" else 1, eps=0.0)
    if fam in ("motion", "motion_ts", "segment"):
        v["warp"], v["K"] = 4, 6
    elif fam in ("motion_depth", "motion_ts_depth"):
        v["warp"], v["K"] = 7, 8
    v.update(overrides)
    return v


def batched_entries():
    return [e for es in BATCHED.values() for e in es]


# ---- the representation, warp and gradient entries ---------------------------------------------------------------------
QUERY_OF = {"evk_voxel_negpos_f32": "evk_voxel_workspace_bytes", "evk_voxel_aos_f32": "evk_voxel_workspace_bytes",
            "evk_voxel_packed_f32": "evk_voxel_workspace_bytes"}
QUERY_OF.update((e, "evk_cmax_workspace_bytes") for e in (
    "evk_cmax_linvel_variance_f64", "evk_cmax_linvel_variance_f32", "evk_cmax_linvel_objective_f64",
    "evk_cmax_linvel_objective_f32", "evk_cmax_linvel_objective_batch_f64", "evk_cmax_warp_objective_f64",
    "evk_cmax_warp_objective_f32", "evk_cmax_warp_objective_batch_f64", "evk_cmax_linvel_partial_f64",
    "evk_cmax_linvel_partial_f32", "evk_cmax_flow_variance_f32", "evk_iwe_objective_f32", "evk_variance_objective_f32",
    "evk_cmax_peer_tail_f32"))
WORKSPACE_FACTOR = {"evk_voxel_negpos_f32": 2}     # evk.h: 2 * evk_voxel_workspace_bytes(B, H, W, flags)

ACC_FLAG, BILINEAR, CLIP, NEGPOS_TRUTHY = 0x1, 0x2, 0x4, 0x8
TS_REVERSE, TS_RAW = 0x80, 0x1000
WINDOW_PAIRS, WINDOW_NEGPOS, AUTO_SPAN = 0x100000, 0x400000, 0x200000
AUTO, GLOBAL_RED, VECTOR_RED, SMEM_TILE, WARP_AGG = (v << 8 for v in (0, 1, 2, 3, 4))   # AUTO only below 2^20 events
CMAX_WANT_GRAD = 0x10


# entries that cannot be captured in a CUDA graph by design, with the reason (none today)
NOT_CAPTURABLE = {}


def _events(rng, n, H, W, outside=3):
    """candidate_checks.draw's events with t = d - d[0] (sorted, from 0), the last `outside` of them moved beyond the
    right edge (index errors)"""
    x, y, d, p, _ = draw(rng, n + outside, H + 1, W + 1)
    x[n:] += W + 2.0
    return x, y, (d - d[0]).astype(np.float32), p


def _voxel(entry, tag, flags, B, H, W, n, seed):
    rng = np.random.default_rng(seed)
    x, y, t, p = _events(rng, n, H, W)
    m = len(x)
    v = dict(n=m, t0=0.0, dt=1.0, B=B, H=H, W=W, flags=flags, oob=Out(8, np.uint64, ACCUMULATE))
    grids = 2 if entry == "evk_voxel_negpos_f32" else 1
    mode = ACCUMULATE if flags & ACC_FLAG else OVERWRITE
    out = Out(grids * B * H * W * 4, np.float32, mode)
    if entry == "evk_voxel_aos_f32":
        v.update(ev=np.column_stack((x, y, t, p)).astype(np.float32), out=out)
    elif entry == "evk_voxel_packed_f32":
        v.update(x=np.floor(x).astype(np.int16), y=np.floor(y).astype(np.int16), t=t.astype(np.float64) + 100.0,
                 p=rng.integers(0, 2, m).astype(np.uint8), t_first=100.0, t_last=100.0 + float(t[-1]), out=out)
    else:
        v.update(x=x, y=y, t=t, p=p)
        v["out_pos_neg" if grids == 2 else "out"] = out
    return Case(entry, tag, v, rtol=2e-5)


def _windows(tag, flags, B, H, W, sizes, seed):
    rng = np.random.default_rng(seed)
    n = int(sum(sizes))
    x, y, t, p = _events(rng, n, H, W, outside=0)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    nw = len(sizes)
    if flags & WINDOW_PAIRS:
        off = np.column_stack((off[:-1], off[1:])).ravel()
    grids = 2 if flags & WINDOW_NEGPOS else 1
    v = dict(x=x, y=y, t=t, p=p, offsets=off, n_windows=nw, n_events_hint=n, B=B, H=H, W=W, flags=flags,
             out=Out(nw * grids * B * H * W * 4, np.float32), oob=Out(8, np.uint64, ACCUMULATE))
    return Case("evk_voxel_windows_f32", tag, v, rtol=2e-5)


def _single_window(sh, H, W, n, seed):
    """the single-window contrast entries, their sharded event pass and its peer tail at world = 1, the image-space tails
    and the derivative helpers on an H x W sensor"""
    rng = np.random.default_rng(seed + 2)
    x, y, t, p = _events(rng, n, H, W)
    m = len(x)
    Hc, Wc = H + 1, W + 1
    f64 = np.float64
    ev64 = dict(x=x.astype(f64), y=y.astype(f64), t=t.astype(f64), p=p.astype(f64), t_ref=0.0)
    ev32 = dict(x=x, y=y, t_rel=t, p=p)
    common = dict(n=m, p_scale=1.0, Hm=H, Wm=W, Hs=H, Ws=W, sigma=1.0, flags=CMAX_WANT_GRAD, objective=0, obj_param=2.0,
                  iwe_out=Out(Hc * Wc * 4, np.float32), diwe_out=Out(2 * Hc * Wc * 4, np.float32))
    vel = dict(vx=30.0, vy=-20.0)
    cases = []
    for suf, ev in (("f64", ev64), ("f32", ev32)):
        cases.append(Case("evk_cmax_linvel_variance_" + suf, sh, dict(common, **ev, **vel, result=Out(8 * 8, f64)), rtol=2e-5))
        for name, obj in (("variance", 0), ("sos", 1), ("soe", 2), ("moa", 3), ("isoa", 4), ("sosa", 5)):
            cases.append(Case("evk_cmax_linvel_objective_" + suf, "%s-%s" % (sh, name), dict(
                common, **ev, **vel, objective=obj, result=Out(12 * 8, f64)), rtol=2e-5))
        model = Host([(W - 1) / 2.0, (H - 1) / 2.0, 3.0])
        cases.append(Case("evk_cmax_warp_objective_" + suf, sh + "-rotation", dict(
            {k: v for k, v in common.items() if k != "diwe_out"}, **ev, warp=1, model=model, result=Out(16 * 8, f64)),
            rtol=2e-5))
        cases.append(Case("evk_cmax_linvel_partial_" + suf, sh, dict(
            {k: v for k, v in common.items() if k not in ("iwe_out", "diwe_out")}, **ev, **vel,
            images_out=Out(3 * Hc * Wc * 4, np.float32), oob_out=Out(8, np.uint64)), rtol=2e-5))
    for J, sig in ((1, 1.0), (32, 0.0), (7, 9.0)):
        cases.append(Case("evk_cmax_linvel_objective_batch_f64", "%s-J%d-sigma%g" % (sh, J, sig), dict(
            common, **ev64, params_host=Host(rng.uniform(-40, 40, (J, 2))), n_params=J, sigma=sig,
            results=Out(12 * 8 * J, f64)), rtol=2e-5))
        rot = np.column_stack((np.full(J, (W - 1) / 2.0), np.full(J, (H - 1) / 2.0), rng.uniform(-5, 5, J)))
        cases.append(Case("evk_cmax_warp_objective_batch_f64", "%s-J%d-sigma%g" % (sh, J, sig), dict(
            common, **ev64, warp=1, models_host=Host(rot), n_models=J, sigma=sig, results=Out(16 * 8 * J, f64)), rtol=2e-5))
    cases.append(Case("evk_cmax_flow_variance_f32", sh, dict(
        common, flags=0, x=x, y=y, t=t, p=p, flow=rng.uniform(-20, 20, (2, H, W)).astype(np.float32), t0=0.0,
        result=Out(8 * 8, f64)), rtol=2e-5))
    iwe = rng.random((Hc, Wc)).astype(np.float32)
    diwe = rng.uniform(-1, 1, (2, Hc, Wc)).astype(np.float32)
    tail = dict(iwe=iwe, diwe=diwe, Hc=Hc, Wc=Wc, Hs=H, Ws=W, sigma=1.0, flags=CMAX_WANT_GRAD)
    for name, obj in (("variance", 0), ("sos", 1), ("sosa", 5)):
        cases.append(Case("evk_iwe_objective_f32", "%s-%s" % (sh, name), dict(tail, objective=obj, obj_param=2.0,
                                                                            result=Out(12 * 8, f64)), rtol=2e-5))
    cases.append(Case("evk_variance_objective_f32", sh, dict(tail, result=Out(8 * 8, f64)), rtol=2e-5))
    planes = np.concatenate([iwe.ravel(), diwe.ravel()]).astype(np.float32)
    cases.append(Case("evk_cmax_peer_tail_f32", sh + "-world1", dict(
        images=planes, oob_count=np.array([3], np.uint64), peer_images=DevicePointers("images"),
        peer_oob=DevicePointers("oob_count"), world=1, Hc=Hc, Wc=Wc, Hs=H, Ws=W, sigma=1.0, flags=CMAX_WANT_GRAD,
        result=Out(8 * 8, f64)), rtol=2e-5))
    K = 2
    jx, jy = rng.uniform(-1, 1, (K, m)).astype(np.float32), rng.uniform(-1, 1, (K, m)).astype(np.float32)
    for name, fl in (("plain", 0), ("clip", CLIP), ("acc", ACC_FLAG)):
        mode = ACCUMULATE if fl & ACC_FLAG else OVERWRITE
        cases.append(Case("evk_image_drv_f32", "%s-%s" % (sh, name), dict(
            x=x, y=y, p=p, jx=jx, jy=jy, K=K, n=m, Himg=Hc, Wimg=Wc, clipx=float(W), clipy=float(H), flags=fl,
            img=Out(Hc * Wc * 4, np.float32, mode), dimg=Out(K * Hc * Wc * 4, np.float32, mode),
            oob=Out(8, np.uint64, ACCUMULATE)), rtol=2e-5))
    px, py = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    cases.append(Case("evk_splat_drv_idx_f32", sh, dict(
        px=px, py=py, dx=(x - px).astype(np.float32), dy=(y - py).astype(np.float32), w1=jx, w2=jy, K=K, n=m, H=H, W=W,
        dimg=Out(K * H * W * 4, np.float32, ACCUMULATE), oob=Out(8, np.uint64, ACCUMULATE)), rtol=2e-5))
    return cases


def simple_cases(seed=100):
    cases = []
    for H, W, n in ((2, 2, 50), (37, 53, 3000), (180, 240, 20000)):
        sh = "%dx%d" % (H, W)
        cases += _single_window(sh, H, W, n, seed)
        cases.append(_voxel("evk_voxel_f32", sh + "-auto", AUTO, 5, H, W, n, seed))
        for name, var in (("global", GLOBAL_RED), ("vector", VECTOR_RED), ("smem", SMEM_TILE)):
            cases.append(_voxel("evk_voxel_f32", "%s-%s" % (sh, name), var, 5, H, W, n, seed))
            cases.append(_voxel("evk_voxel_f32", "%s-%s-acc" % (sh, name), var | ACC_FLAG, 5, H, W, n, seed))
        cases.append(_voxel("evk_voxel_f32", sh + "-global-bilinear", GLOBAL_RED | BILINEAR, 5, H, W, n, seed))
        cases.append(_voxel("evk_voxel_f32", sh + "-vector-bilinear-acc", VECTOR_RED | BILINEAR | ACC_FLAG, 5, H, W, n, seed))
        cases.append(_voxel("evk_voxel_f32", sh + "-vector-autospan", VECTOR_RED | AUTO_SPAN, 3, H, W, n, seed))
        for name, var in (("global", GLOBAL_RED), ("vector", VECTOR_RED)):
            cases.append(_voxel("evk_voxel_negpos_f32", "%s-%s" % (sh, name), var, 5, H, W, n, seed))
            cases.append(_voxel("evk_voxel_negpos_f32", "%s-%s-truthy-acc" % (sh, name), var | NEGPOS_TRUTHY | ACC_FLAG, 5, H,
                                W, n, seed))
            cases.append(_voxel("evk_voxel_aos_f32", "%s-%s" % (sh, name), var, 5, H, W, n, seed))
            cases.append(_voxel("evk_voxel_packed_f32", "%s-%s" % (sh, name), var, 5, H, W, n, seed))
        for name, fl in (("plain", 0), ("pairs", WINDOW_PAIRS), ("negpos", WINDOW_NEGPOS)):
            cases.append(_windows("%s-%s" % (sh, name), fl, 5, H, W, [n // 2, 0, 1, n // 2], seed))
        rng = np.random.default_rng(seed + 1)
        x, y, t, p = _events(rng, n, H, W)
        m = len(x)
        for name, fl in (("nearest", 0), ("bilinear", BILINEAR), ("clip", CLIP), ("bilinear-clip", BILINEAR | CLIP),
                         ("acc", ACC_FLAG), ("bilinear-acc", BILINEAR | ACC_FLAG), ("global", GLOBAL_RED),
                         ("warpagg-clip", WARP_AGG | CLIP), ("smem", SMEM_TILE), ("smem-acc", SMEM_TILE | ACC_FLAG),
                         ("bilinear-vector", BILINEAR | VECTOR_RED)):
            mode = ACCUMULATE if fl & ACC_FLAG else OVERWRITE
            cases.append(Case("evk_image_f32", "%s-%s" % (sh, name), dict(
                x=x, y=y, p=p, n=m, Himg=H, Wimg=W, clipx=W - 1.0, clipy=H - 1.0, flags=fl, fill=0.5,
                out=Out(H * W * 4, np.float32, mode), oob=Out(8, np.uint64, ACCUMULATE)), rtol=2e-5))
        for name, fl in (("plain", 0), ("clip", CLIP), ("acc", ACC_FLAG), ("smem", SMEM_TILE), ("smem-acc", SMEM_TILE | ACC_FLAG)):
            mode = ACCUMULATE if fl & ACC_FLAG else OVERWRITE
            cases.append(Case("evk_count_u32", "%s-%s" % (sh, name), dict(
                x=x, y=y, n=m, Himg=H, Wimg=W, clipx=W - 1.0, clipy=H - 1.0, flags=fl,
                out=Out(H * W * 4, np.uint32, mode), oob=Out(8, np.uint64, ACCUMULATE))))
        for name, fl in (("plain", 0), ("clip", CLIP), ("reverse", TS_REVERSE), ("raw", TS_RAW), ("clip-reverse", CLIP | TS_REVERSE)):
            base = dict(x=x, y=y, t=t, p=p, n=m, t_first=float(t[0]), t_last=float(t[-1]), Himg=H + 1, Wimg=W + 1,
                        clipx=float(W), clipy=float(H), flags=fl)
            img = (H + 1) * (W + 1) * 4
            cases.append(Case("evk_timestamp_image_f32", "%s-%s" % (sh, name), dict(
                base, out_pos=Out(img, np.float32), out_neg=Out(img, np.float32), oob=Out(8, np.uint64, ACCUMULATE)),
                rtol=2e-5))
            cases.append(Case("evk_timestamp_image_counts_f32", "%s-%s" % (sh, name), dict(
                base, out_pos=Out(img, np.float32), out_neg=Out(img, np.float32), cnt_pos=Out(img, np.float32),
                cnt_neg=Out(img, np.float32), oob=Out(8, np.uint64, ACCUMULATE)), rtol=2e-5))
        flow = rng.uniform(-2, 2, (2, H, W)).astype(np.float32)
        cases.append(Case("evk_warp_flow_f32", sh, dict(x=x, y=y, t=t, n=m, flow=flow, H=H, W=W, t0=0.25,
                                                         xw=Out(m * 4, np.float32), yw=Out(m * 4, np.float32))))
        gxw, gyw = rng.uniform(-1, 1, m).astype(np.float32), rng.uniform(-1, 1, m).astype(np.float32)
        cases.append(Case("evk_warp_flow_grad_f32", sh, dict(
            x=x, y=y, t=t, n=m, flow=flow, H=H, W=W, t0=0.25, grad_xw=gxw, grad_yw=gyw, grad_x=Out(m * 4, np.float32),
            grad_y=Out(m * 4, np.float32), grad_t=Out(m * 4, np.float32), grad_flow=Out(2 * H * W * 4, np.float32),
            sum_grad_t=Out(8, np.float64)), rtol=2e-5))
        gimg = rng.uniform(-1, 1, (H, W)).astype(np.float32)
        cases.append(Case("evk_image_grad_f32", sh + "-bilinear", dict(
            x=x, y=y, p=p, n=m, Himg=H, Wimg=W, clipx=W - 1.0, clipy=H - 1.0, flags=BILINEAR, grad_img=gimg,
            grad_x=Out(m * 4, np.float32), grad_y=Out(m * 4, np.float32), grad_p=Out(m * 4, np.float32))))
        cases.append(Case("evk_image_grad_f32", sh + "-nearest-clip", dict(
            x=x, y=y, p=p, n=m, Himg=H, Wimg=W, clipx=W - 1.0, clipy=H - 1.0, flags=CLIP, grad_img=gimg,
            grad_x=None, grad_y=None, grad_p=Out(m * 4, np.float32))))
        Hc, Wc = H + 1, W + 1
        for name, fl in (("plain", 0), ("clip-reverse", CLIP | TS_REVERSE)):
            cases.append(Case("evk_timestamp_image_grad_f32", "%s-%s" % (sh, name), dict(
                x=x, y=y, t=t, p=p, n=m, t_first=float(t[0]), t_last=float(t[-1]), Himg=Hc, Wimg=Wc, clipx=float(W),
                clipy=float(H), flags=fl, grad_pos=rng.uniform(-1, 1, (Hc, Wc)).astype(np.float32),
                grad_neg=rng.uniform(-1, 1, (Hc, Wc)).astype(np.float32), out_pos=rng.random((Hc, Wc)).astype(np.float32),
                out_neg=rng.random((Hc, Wc)).astype(np.float32), cnt_pos=(1 + rng.random((Hc, Wc))).astype(np.float32),
                cnt_neg=(1 + rng.random((Hc, Wc))).astype(np.float32), grad_x=Out(m * 4, np.float32),
                grad_y=Out(m * 4, np.float32), grad_t=Out(m * 4, np.float32), sums=Out(16, np.float64)), rtol=2e-5))
        sizes = [n // 2, 0, 1, n // 2]
        ends = np.cumsum(sizes)
        pairs = np.column_stack((ends - sizes, ends)).astype(np.int64).ravel()
        xs, ys, ts, ps = _events(rng, int(ends[-1]), H, W, outside=0)
        nw = len(sizes)
        cases.append(Case("evk_voxel_grad_f32", sh + "-windows", dict(
            x=xs, y=ys, t=ts, p=ps, n=len(xs), pairs=pairs, n_windows=nw, B=5, H=H, W=W, flags=0,
            grad_out=rng.uniform(-1, 1, (nw, 5, H, W)).astype(np.float32), grad_p=Out(len(xs) * 4, np.float32),
            grad_t=Out(len(xs) * 4, np.float32)), rtol=2e-5))
        img = rng.random((H, W)).astype(np.float32)
        cases.append(Case("evk_gaussian_blur_f32", sh, dict(img=img, H=H, W=W, sigma=1.5, out=Out(H * W * 4, np.float32),
                                                             tmp=Out(H * W * 4, np.float32, SCRATCH))))
        img64 = rng.random((H, W))
        cases.append(Case("evk_gather_bilinear_f64", sh, dict(
            x=x.astype(np.float64) - 0.5, y=y.astype(np.float64) - 0.5, n=m, img=img64, H=H, W=W,
            out=Out(m * 8, np.float64), oob=Out(8, np.uint64, ACCUMULATE))))
        px, py = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
        cases.append(Case("evk_splat_idx_f32", sh, dict(
            px=px, py=py, dx=(x - px).astype(np.float32), dy=(y - py).astype(np.float32), w=p, n=m, H=H, W=W,
            img=Out(H * W * 4, np.float32, ACCUMULATE), oob=Out(8, np.uint64, ACCUMULATE)), rtol=2e-5))
    for n in (1, 2, 1000, 100003):
        xr = np.random.default_rng(seed + n).standard_normal(n).astype(np.float32)
        cases.append(Case("evk_robust_norm_f32", "n%d" % n, dict(
            x=xr, n=n, k_low=1 + round(0.01 * (n - 1)), k_top=1 + round(0.99 * (n - 1)), out=Out(n * 4, np.float32),
            t_min_max=Out(8, np.float32))))
    return cases


SIMPLE = sorted({c.entry for c in simple_cases()})
