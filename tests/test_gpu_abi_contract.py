"""The memory and stream contract of every device entry with a case in tests/abi_contract_cases.py, on the GPU.

For each case:
  - bounds: the workspace and every output share one allocation, each flanked by 4 KiB guard bands of a fixed byte;
    each region is placed once on a 256-byte boundary and once ending as close to the next boundary as its alignment
    allows, and after the call no guard byte may have changed;
  - outputs fully written: overwritten outputs start as 0xFF bytes (NaN in f32 and f64) and must equal the clean run,
    NaN positions included; accumulated outputs start as a known image and out - base must equal the clean run;
  - scratch independence: workspaces of 0x00, 0xFF, 0x7F and random bytes all give the clean run's outputs, and a large
    call followed by a small one on the same uncleared buffer gives the small one's clean outputs;
  - the inputs are never written;
  - stream and synchronisation: after an eager warm-up the call is captured in a CUDA graph on a side stream in global
    capture mode (a synchronisation, a launch on another stream or an allocation inside the library invalidates the
    capture), and a replay over poisoned outputs and workspace reproduces the eager outputs;
  - refusals write nothing (the batched losses): a NaN blur sigma, a workspace one byte short and one 128 bytes off its
    alignment leave every output, the workspace and the guards byte-identical.  These are refusals that stay in bounds
    even if an entry wrongly accepted them; the limit refusals of tests/test_abi_contract_cpu.py (batch past its cap
    and the like) would, if wrongly accepted, launch past the ends of real buffers, so they are made only with
    placeholder pointers on a machine without a GPU;
  - anchors: one case of each batched family against its f64 reference in tests/*_reference.py, at the family's
    tolerance, so that the cases compare the library with the reference and not only with itself.
"""
import ctypes

import numpy as np
import pytest
import torch

import abi_contract_cases as C

pytestmark = pytest.mark.gpu

GUARD = 4096
PATTERN = 0xA5
E_ARG, E_WORKSPACE = -1, -3


@pytest.fixture(scope="module")
def L():
    from event_utils_b200 import _lib
    return _lib.lib()


def _align(v, a):
    return (v + a - 1) // a * a


class Layout:
    """the workspace and the outputs of a case in one guarded allocation"""

    def __init__(self, case, ws_bytes, tail):
        regions = [("workspace", ws_bytes, 256)] if ws_bytes else []
        regions += [(k, o.nbytes, 16) for k, o in case.outputs().items()]
        off, self.at = GUARD, {}
        for name, nb, al in regions:
            start = _align(off, 256)
            if tail and nb % 256:
                start += (256 - nb % 256) // al * al       # end as close to the next 256-byte boundary as `al` allows
            self.at[name] = (start, nb)
            off = start + nb + GUARD
        self.total = _align(off, 256)
        self.buf = torch.empty(self.total, dtype=torch.uint8, device="cuda")
        guard = torch.ones(self.total, dtype=torch.bool)
        for s, nb in self.at.values():
            guard[s:s + nb] = False
        self.guard = guard.cuda()

    def view(self, name):
        s, nb = self.at[name]
        return self.buf[s:s + nb]

    def ptr(self, name, offset=0):
        return self.buf.data_ptr() + self.at[name][0] + offset if name in self.at else None

    def guards_intact(self):
        return bool((self.buf[self.guard] == PATTERN).all())


def _fill(t, how, gen):
    if how == "random":
        t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device=t.device, generator=gen))
    else:
        t.fill_(how)


class Runner:
    def __init__(self, L, case):
        self.L, self.case = L, case
        self.inputs = {}
        for k, v in case.values.items():
            if isinstance(v, np.ndarray):
                self.inputs[k] = (v, torch.from_numpy(np.ascontiguousarray(v)).cuda())
        self.tables = {k: (ctypes.c_void_p * len(v.names))(*[self.inputs[n][1].data_ptr() for n in v.names])
                       for k, v in case.values.items() if isinstance(v, C.DevicePointers)}
        self.ws_bytes = case.workspace_bytes(L)
        self.gen = torch.Generator(device="cuda")
        self.gen.manual_seed(1234)
        self.base = {}
        for k, o in case.outputs().items():
            if o.mode == C.ACCUMULATE:      # small integers: base + clean rounds like clean alone, to one ulp of the sum
                n = o.nbytes // o.dtype.itemsize
                self.base[k] = np.random.default_rng(7).integers(0, 4, n).astype(o.dtype)

    def args(self, lay, stream, ws_offset=0, ws_bytes=None, over=None):
        out = []
        for name in C.protos()[self.case.entry]:
            if over and name in over:
                out.append(over[name])
            elif name == "workspace":
                out.append(lay.ptr("workspace", ws_offset))
            elif name == "workspace_bytes":
                out.append(self.ws_bytes if ws_bytes is None else ws_bytes)
            elif name == "stream":
                out.append(ctypes.c_void_p(stream))
            elif name in self.inputs:
                out.append(self.inputs[name][1].data_ptr())
            elif name in self.tables:
                out.append(ctypes.cast(self.tables[name], ctypes.c_void_p))
            elif isinstance(self.case.values.get(name), C.Host):
                out.append(self.case.values[name].arr.ctypes.data)
            elif name in lay.at:
                out.append(lay.ptr(name))
            else:
                out.append(self.case.values[name])
        return out

    def prepare(self, lay, ws_fill, out_fill=0xFF):
        lay.buf.fill_(PATTERN)
        if "workspace" in lay.at:
            _fill(lay.view("workspace"), ws_fill, self.gen)
        for k, o in self.case.outputs().items():
            if o.mode == C.ACCUMULATE:
                lay.view(k).copy_(torch.from_numpy(self.base[k].view(np.uint8)).cuda())
            else:
                _fill(lay.view(k), out_fill, self.gen)

    def call(self, lay, stream=None, **kw):
        s = torch.cuda.current_stream().cuda_stream if stream is None else stream
        return getattr(self.L, self.case.entry)(*self.args(lay, s, **kw))

    def outputs(self, lay):
        res = {}
        for k, o in self.case.compared().items():
            a = lay.view(k).cpu().numpy().view(o.dtype).copy()
            if o.mode == C.ACCUMULATE:
                a = a - self.base[k]
            res[k] = a
        return res

    def run(self, lay, ws_fill, out_fill=0xFF):
        self.prepare(lay, ws_fill, out_fill)
        rc = self.call(lay)
        torch.cuda.synchronize()
        assert rc == 0, "%s: rc %d (%s)" % (self.case.id, rc, self.L.evk_last_error())
        assert lay.guards_intact(), "%s: a guard band changed (write outside the workspace or an output)" % self.case.id
        return self.outputs(lay)

    def inputs_unchanged(self):
        for k, (a, t) in self.inputs.items():
            assert np.array_equal(t.cpu().numpy().view(np.uint8), np.ascontiguousarray(a).view(np.uint8)), \
                "%s: input %s was written" % (self.case.id, k)


def assert_same(case, got, want, what):
    for k, w in want.items():
        g = got[k]
        o = case.outputs()[k]
        if o.dtype.kind != "f":
            assert np.array_equal(g, w), "%s %s: %s differs" % (case.id, what, k)
            continue
        nan_g, nan_w = np.isnan(g), np.isnan(w)
        assert (nan_g == nan_w).all(), "%s %s: %s has NaN at %d positions where the clean run has none (or the reverse)" % (
            case.id, what, k, int((nan_g != nan_w).sum()))
        fin = ~nan_w
        if not fin.any():
            continue
        if case.rtol == 0 and o.mode == C.OVERWRITE:
            assert np.array_equal(g[fin].view(np.uint8), w[fin].view(np.uint8)), "%s %s: %s differs" % (case.id, what, k)
            continue
        scale = float(np.abs(w[fin]).max())
        if o.mode == C.ACCUMULATE:
            scale += 4.0
        tol = max(case.rtol, 4 * float(np.finfo(o.dtype).eps)) * max(scale, 1e-30)
        err = float(np.abs(g[fin].astype(np.float64) - w[fin]).max())
        assert err <= tol, "%s %s: %s max err %.3e > %.3e" % (case.id, what, k, err, tol)


CASES = C.batched_cases() + C.simple_cases()
assert not set(C.NOT_CAPTURABLE) - {c.entry for c in CASES}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_bounds_full_writes_and_scratch_independence(L, case):
    r = Runner(L, case)
    clean = r.run(Layout(case, r.ws_bytes, False), 0x00, out_fill=0x00)
    for tail in (False, True):
        lay = Layout(case, r.ws_bytes, tail)
        for fill in (0x00, 0xFF, 0x7F, "random"):
            got = r.run(lay, fill)
            assert_same(case, got, clean, "(workspace %s, %s placement)" % (fill, "tail" if tail else "head"))
    r.inputs_unchanged()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_graph_capture_on_a_side_stream(L, case):
    if case.entry in C.NOT_CAPTURABLE:
        pytest.skip(C.NOT_CAPTURABLE[case.entry])
    r = Runner(L, case)
    lay = Layout(case, r.ws_bytes, False)
    eager = r.run(lay, 0x00)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rc = r.call(lay, side.cuda_stream)          # eager warm-up on the side stream
    torch.cuda.synchronize()
    assert rc == 0
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side, capture_error_mode="global"):
        rc = r.call(lay, side.cuda_stream)
    assert rc == 0, "%s: rc %d under capture (%s)" % (case.id, rc, L.evk_last_error())
    r.prepare(lay, "random")
    g.replay()
    torch.cuda.synchronize()
    assert lay.guards_intact(), case.id
    assert_same(case, r.outputs(lay), eager, "(graph replay)")
    del g


@pytest.mark.parametrize("case", C.batched_cases(), ids=lambda c: c.id)
def test_refusals_write_nothing(L, case):
    """the batched losses, whose workspace is required (the voxel, image and warp entries also run without one)"""
    r = Runner(L, case)
    lay = Layout(case, r.ws_bytes, False)
    r.prepare(lay, "random")
    before = lay.buf.clone()
    refusals = [dict(ws_bytes=r.ws_bytes - 1), dict(ws_offset=128)]
    names = C.protos()[case.entry]
    for key in ("sigma", "blur_sigma"):
        if key in names:
            refusals.append(dict(over={key: float("nan")}))
    for kw in refusals:
        if kw.get("ws_bytes", 0) < 0:
            continue
        rc = r.call(lay, **kw)
        torch.cuda.synchronize()
        assert rc in (E_ARG, E_WORKSPACE), "%s %s: rc %d" % (case.id, kw, rc)
        assert torch.equal(lay.buf, before), "%s %s: a refused call wrote memory" % (case.id, kw)


def _family_pairs():
    """per batched family and entry kind, the case with the largest workspace and the one with the smallest"""
    by = {}
    for c in C.batched_cases():
        by.setdefault(c.entry, []).append(c)
    return [(e, cs) for e, cs in by.items() if len(cs) > 1]


@pytest.mark.parametrize("entry,cases", _family_pairs(), ids=lambda v: v if isinstance(v, str) else "")
def test_large_then_small_call_on_one_uncleared_workspace(L, entry, cases):
    """what the torch layer does with its cached scratch (_lib.scratch): a small call right after a large one on the
    same workspace, nothing cleared in between"""
    runners = [Runner(L, c) for c in cases]
    big = max(runners, key=lambda r: r.ws_bytes)
    for small in runners:
        if small is big:
            continue
        fresh = small.run(Layout(small.case, small.ws_bytes, False), 0x00, out_fill=0x00)
        ws = torch.zeros(big.ws_bytes + 256, dtype=torch.uint8, device="cuda")
        lay_big = Layout(big.case, 0, False)
        big.prepare(lay_big, 0x00)
        ws_ptr = _align(ws.data_ptr(), 256)
        rc = getattr(L, entry)(*big.args(lay_big, torch.cuda.current_stream().cuda_stream, over={"workspace": ws_ptr}))
        assert rc == 0
        lay_small = Layout(small.case, 0, False)
        small.prepare(lay_small, 0x00)
        args = small.args(lay_small, torch.cuda.current_stream().cuda_stream,
                          over={"workspace": ws_ptr, "workspace_bytes": small.ws_bytes})
        rc = getattr(L, entry)(*args)
        torch.cuda.synchronize()
        assert rc == 0
        assert_same(small.case, small.outputs(lay_small), fresh, "(after %s on the same workspace)" % big.case.tag)


def _anchor_cases():
    want = {"evk_cmax_flow_objective_f32", "evk_flow_timestamp_objective_f32", "evk_cmax_motion_objective_f32",
            "evk_motion_timestamp_objective_f32", "evk_cmax_motion_segment_f32", "evk_cmax_grid_flow_objective_f32",
            "evk_cmax_depth_grid_objective_f32"}
    return [c for c in C.batched_cases() if c.entry in want and c.tag == "37x53-skew-J1-M2"]


def _reference(case):
    """f (B or B M), and the images (the IWEs, or T and C) of the f64 reference of the case's family"""
    import depth_grid_reference
    import flow_objective_reference
    import flow_timestamp_reference
    import grid_flow_reference
    import planar_motion_reference
    v = case.values
    x, y, d, p, off, H, W, s = v["x"], v["y"], v["t_rel"], v["p"], v["offsets"], v["H"], v["W"], v["sigma"]
    dbl = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    e, centre = case.entry, (v["cx"], v["cy"])
    if e == "evk_cmax_flow_objective_f32":
        f, iwe, _ = flow_objective_reference.reference(x, y, d, p, off, dbl(v["flow"]), s, "variance")
        return f, {"iwe_out": iwe}
    if e == "evk_flow_timestamp_objective_f32":
        f, T, Cc = flow_timestamp_reference.reference(x, y, d, v["tau"], p, off, dbl(v["flow"]), s)
        return f, {"ts_out": T, "cnt_out": Cc}
    if e == "evk_cmax_motion_objective_f32":
        f, iwe = planar_motion_reference.contrast("affine", x, y, d, p, off, dbl(v["params"]), s, "variance",
                                                  img_size=(H, W), centre=centre)
        return f, {"iwe_out": iwe}
    if e == "evk_motion_timestamp_objective_f32":
        out = planar_motion_reference.timestamp("affine", x, y, d, v["tau"], p, off, dbl(v["params"]), s, img_size=(H, W),
                                                centre=centre)
        return out[0], {"ts_out": out[1], "cnt_out": out[2]}
    if e == "evk_cmax_motion_segment_f32":
        # image (b, m) is the motion loss's on p * weights[:, m] under params[:, m] (evk.h)
        M = v["n_models"]
        outs = [planar_motion_reference.contrast("affine", x, y, d, (p * v["weights"][:, m]).astype(np.float32), off,
                                                 dbl(v["params"][:, m]), s, "variance", img_size=(H, W), centre=centre)
                for m in range(M)]
        return torch.stack([o[0] for o in outs], 1), {"iwe_out": torch.stack([o[1] for o in outs], 1)}
    if e == "evk_cmax_grid_flow_objective_f32":
        f, iwe = grid_flow_reference.reference(x, y, d, p, off, dbl(v["grid_flow"]), H, W, s, "variance")[:2]
        return f, {"iwe_out": iwe}
    m = v["motion"]
    intr = (m[0, 6], m[0, 7], v["cx"], v["cy"])
    f, iwe = depth_grid_reference.contrast(x, y, d, p, off, dbl(v["inv_depth_grid"]), m[:, :6], intr, s, "variance",
                                           img_size=(H, W))[:2]
    return f, {"iwe_out": iwe}


@pytest.mark.parametrize("case", _anchor_cases(), ids=lambda c: c.id)
def test_anchor_to_the_f64_reference(L, case):
    """the clean run of one case per family against its f64 reference: f and the images to 1e-5 of their largest
    magnitude, the tolerance of the family's own tests"""
    from conftest import assert_close_to_max
    r = Runner(L, case)
    got = r.run(Layout(case, r.ws_bytes, False), "random")
    f, images = _reference(case)
    f = np.asarray(f.detach().numpy() if hasattr(f, "detach") else f, np.float64).ravel()
    assert_close_to_max(got["f_out"], f, 1e-5, case.id + " f")
    for k, img in images.items():
        img = np.asarray(img.detach().numpy() if hasattr(img, "detach") else img, np.float64)
        assert_close_to_max(got[k].reshape(img.shape), img, 1e-5, "%s %s" % (case.id, k))
