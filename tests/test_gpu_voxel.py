"""Parity of the CUDA voxel path (through the python drop-in layer and the C ABI) with the
oracle and with the golden vectors of the real reference."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import assert_close_to_max, golden, make_events

pytestmark = pytest.mark.gpu

import os as _os

# the routed kernel spins on inter-SM queues; its in-kernel watchdog turns a protocol stall into a RuntimeError instead of a
# hang.  tools/try_routed.py is the stand-alone gate; EVK_TEST_ROUTED=0 keeps the variant out of this suite
ROUTED = ["routed"] if _os.environ.get("EVK_TEST_ROUTED", "1") != "0" else []
VARIANTS = ["global_red", "vector_red", "smem_cache"] + ROUTED + [None]


@pytest.fixture(autouse=True)
def _reset_variant():
    import event_utils_b200 as eu
    yield
    eu.config.variant = None
    eu.config.check_index_errors = True


def dev(*arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


@pytest.mark.parametrize("variant", VARIANTS)
def test_golden_cases(variant):
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    eu.config.variant = variant
    g = golden("voxel_torch")
    for tag in "abcde":
        H, W = (int(v) for v in g[tag + "_HW"])
        x, y, t, p = dev(g[tag + "_x"], g[tag + "_y"], g[tag + "_t"], g[tag + "_p"])
        out = events_to_voxel_torch(x, y, t, p, int(g[tag + "_B"]), sensor_size=(H, W))
        assert out.is_cuda and out.dtype == torch.float32 and out.shape == g[tag + "_out"].shape
        assert_close_to_max(out.cpu().numpy(), g[tag + "_out"], 1e-5, tag)
    # integer-valued weights -> bit exact (case b: ps == 1, integer coordinates)
    H, W = (int(v) for v in g["b_HW"])
    x, y, t, p = dev(g["b_x"], g["b_y"], g["b_t"], g["b_p"])
    out = events_to_voxel_torch(x, y, t, p, int(g["b_B"]), sensor_size=(H, W)).cpu().numpy()
    assert abs(out.sum() - g["b_out"].sum()) <= 1e-3


@pytest.mark.parametrize("variant", VARIANTS)
def test_negative_wrap_nan_and_oob(variant):
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    eu.config.variant = variant
    g = golden("voxel_torch")
    x, y, t, p = dev(g["neg_x"], g["neg_y"], g["neg_t"], g["neg_p"])
    out = events_to_voxel_torch(x, y, t, p, 3, sensor_size=(4, 6)).cpu().numpy()
    assert_close_to_max(out, g["neg_out"], 1e-6)
    x, y, t, p = dev(g["nan_x"], g["nan_y"], g["nan_t"], g["nan_p"])
    out = events_to_voxel_torch(x, y, t, p, 3, sensor_size=(4, 6)).cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(g["nan_out"]))
    with pytest.raises(IndexError):
        events_to_voxel_torch(*dev(np.float32([6.0, 1.0]), np.float32([0, 0]), np.float32([0, 1]), np.float32([1, 1])), 2, sensor_size=(4, 6))
    with pytest.raises(AssertionError):
        events_to_voxel_torch(*dev(np.float32([1.0, 1.0]), np.float32([0]), np.float32([0, 1]), np.float32([1, 1])), 2)
    with pytest.raises(RuntimeError):  # f64 polarities: the reference's dtype mismatch
        events_to_voxel_torch(*dev(np.float32([1.0, 1.0]), np.float32([0, 0]), np.float32([0, 1]), np.float64([1, 1])), 2)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n,B,H,W,pol", [(200000, 5, 260, 346, "pm1"), (100003, 7, 180, 240, "real"),
                                         (50001, 4, 33, 47, "real"), (77777, 1, 20, 20, "pm1"), (5, 5, 8, 8, "pm1")])
def test_vs_oracle(oracle, variant, n, B, H, W, pol):
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    eu.config.variant = variant
    x, y, t, p = make_events(n + B, n, H, W, pol=pol)
    ref = oracle.voxel_f32(x, y, t, p, B, (H, W))
    out = events_to_voxel_torch(*dev(x, y, t, p), B, sensor_size=(H, W)).cpu().numpy()
    assert_close_to_max(out, ref, 1e-5)
    if pol == "pm1":
        # temporal weights sum to one: the grid total equals the polarity total
        assert abs(float(out.astype(np.float64).sum()) - float(p.astype(np.float64).sum())) <= 1e-4 * n ** 0.5 + 1e-3


def test_count_weights_bit_exact(oracle):
    """integer weights at bin centres only (B=1 => every weight is p*NaN? no: dt*(0)=0 -> w=1)."""
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    x, y, t, p = make_events(9, 300000, 64, 64, pol="ones")
    out = events_to_voxel_torch(*dev(x, y, t, p), 1, sensor_size=(64, 64)).cpu().numpy()
    ref = oracle.voxel_f32(x, y, t, p, 1, (64, 64))
    assert np.array_equal(out, ref)
    assert out.sum() == 300000


def test_unaligned_slices_and_aos(oracle):
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    x, y, t, p = make_events(10, 100010, 100, 120, pol="real")
    X, Y, T, P = dev(x, y, t, p)
    for off in (1, 2, 3, 5):
        sl = slice(off, 100000 + off)
        ref = oracle.voxel_f32(x[sl], y[sl], t[sl], p[sl], 5, (100, 120))
        out = events_to_voxel_torch(X[sl], Y[sl], T[sl], P[sl], 5, sensor_size=(100, 120)).cpu().numpy()
        assert_close_to_max(out, ref, 1e-5, "offset %d" % off)
    # different misalignment per array -> scalar-load kernel
    ref = oracle.voxel_f32(x[1:1001], y[2:1002], t[3:1003], p[0:1000], 5, (100, 120))
    out = events_to_voxel_torch(X[1:1001], Y[2:1002], T[3:1003], P[0:1000], 5, sensor_size=(100, 120)).cpu().numpy()
    assert_close_to_max(out, ref, 1e-5)
    # columns of an (N,4) tensor: the AoS kernel
    ev = torch.stack((X, Y, T, P), dim=1).contiguous()
    from event_utils_b200.representations import _events as E
    assert E.aos_base(ev[:, 0], ev[:, 1], ev[:, 2], ev[:, 3]) is not None
    ref = oracle.voxel_f32(x, y, t, p, 5, (100, 120))
    out = events_to_voxel_torch(ev[:, 0], ev[:, 1], ev[:, 2], ev[:, 3], 5, sensor_size=(100, 120)).cpu().numpy()
    assert_close_to_max(out, ref, 1e-5)


def test_host_inputs_pipeline(oracle):
    """CPU tensors in -> chunked H2D pipeline -> CPU tensor out (the reference's calling convention)."""
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    x, y, t, p = make_events(11, 300000, 180, 240)
    out = events_to_voxel_torch(*(torch.from_numpy(a) for a in (x, y, t, p)), 5)
    assert not out.is_cuda and out.shape == (5, 180, 240)
    assert_close_to_max(out.numpy(), oracle.voxel_f32(x, y, t, p, 5, (180, 240)), 1e-5)
    # numpy in (the reference fails on numpy, base_dataset.py:448; we accept it)
    out = events_to_voxel_torch(x, y, t, p, 5)
    assert_close_to_max(out.numpy(), oracle.voxel_f32(x, y, t, p, 5, (180, 240)), 1e-5)
    # integer coordinates and integer timestamps
    xi, yi = x.astype(np.int64), y.astype(np.int64)
    ti = (t * 1e6).astype(np.int64)
    out = events_to_voxel_torch(torch.from_numpy(xi), torch.from_numpy(yi), torch.from_numpy(ti), torch.from_numpy(p), 5)
    trel = (ti - ti[0]).astype(np.float32)
    assert_close_to_max(out.numpy(), oracle.voxel_f32(xi, yi, trel, p, 5, (180, 240), t0=0.0, dt=trel[-1]), 1e-5)


def test_hot_pixels(oracle):
    """A stream with hot pixels (2 pixels carry 30 % of the events): every variant, incl. the adaptive
    shared-memory cache that AUTO selects for large N, against the oracle; counts bit exact."""
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch, events_to_voxel_torch
    n, H, W = 2_000_000, 260, 346
    x, y, t, p = make_events(77, n, H, W, pol="ones")
    rng = np.random.default_rng(78)
    hot = rng.random(n) < 0.3
    x[hot] = np.where(rng.random(hot.sum()) < 0.5, 17.0, 200.0)
    y[hot] = np.where(x[hot] == 17.0, 33.0, 101.0)
    ref = oracle.voxel_f32(x, y, t, p, 1, (H, W))          # B=1: every weight is exactly 1 -> integer counts
    for variant in VARIANTS:
        eu.config.variant = variant
        out = events_to_voxel_torch(*dev(x, y, t, p), 1, sensor_size=(H, W)).cpu().numpy()
        assert np.array_equal(out, ref), variant
    pm = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    ref5 = oracle.voxel_f32(x, y, t, pm, 5, (H, W))
    refp = oracle.voxel_f32(x, y, t, (pm > 0).astype(np.float32), 5, (H, W))
    # the hot cells sum ~3e5 weights of mixed sign in f32: order-dependent beyond 1e-5 there (see
    # test_gpu_image.test_hot_spot_bilinear_and_signed); the bound is the random-walk one
    bound = 2.0 * np.sqrt(0.15 * n) * np.finfo(np.float32).eps * np.abs(refp).max()
    for variant in VARIANTS:
        eu.config.variant = variant
        out = events_to_voxel_torch(*dev(x, y, t, pm), 5, sensor_size=(H, W)).cpu().numpy()
        assert np.abs(out - ref5).max() <= max(bound, 1e-5 * np.abs(ref5).max()), variant
        vp, vn = events_to_neg_pos_voxel_torch(*dev(x, y, t, pm), 5, sensor_size=(H, W))
        assert np.abs(vp.cpu().numpy() - refp).max() <= bound, variant


@pytest.mark.skipif(not ROUTED, reason="EVK_TEST_ROUTED=0")
def test_auto_probe_picks_between_routed_and_vector_red():
    """AUTO with the routed kernel enabled (EVK_VOXEL_ROUTED_MIN, read once at library load -> a subprocess): a device-side
    probe looks at a sample of the stream; unit-polarity uniform streams take the routed kernel, general polarities and
    hot-pixel streams the vector-reduction kernel; the kernel not chosen returns at once.  All three equal the oracle."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = r'''
import sys
import numpy as np, torch
sys.path.insert(0, %r)
from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
from oracle import evk_oracle as O
O.build()
rng = np.random.default_rng(3)
n, H, W = 3_000_000, 260, 346
x = (rng.random(n) * (W - 1)).astype(np.float32); y = (rng.random(n) * (H - 1)).astype(np.float32)
t = np.sort(rng.random(n)).astype(np.float32)
cases = {"unit": (x, y, (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)),
         "general": (x, y, rng.standard_normal(n).astype(np.float32))}
xh, yh = x.copy(), y.copy()
hot = rng.random(n) < 0.2
xh[hot], yh[hot] = 17.0, 33.0
cases["hot"] = (xh, yh, cases["unit"][2])
for name, (cx, cy, cp) in cases.items():
    ref = O.voxel_f32(cx, cy, t, cp, 5, (H, W))
    out = events_to_voxel_torch(*(torch.from_numpy(a).cuda() for a in (cx, cy, t, cp)), 5, sensor_size=(H, W)).cpu().numpy()
    err = np.abs(out - ref).max() / np.abs(ref).max()
    # the hot pixel sums 6e5 signed f32 taps: the sequential f32 oracle itself is ~sqrt(n) eps away from the exact sum
    # (order-dependent, see test_hot_pixels_*), so that case gets the random-walk allowance instead of 1e-5
    assert err <= (2e-4 if name == "hot" else 1e-5), (name, err)
    print(name, "ok %%.2e" %% err)
''' % root
    out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=root,
                         env=dict(os.environ, EVK_VOXEL_ROUTED_MIN="1000000"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert "hot ok" in out.stdout


def test_host_pipeline_pageable_and_pinned(oracle):
    """Host f32 tensors take the chunked H2D pipeline (evk_voxel_host_f32): pinned sources are copied directly, ordinary
    pageable ones -- what the reference's callers hand over -- through pinned bounce buffers filled by host threads.
    9 M events = three 4 M-event chunks (both bounce slots are reused), same grid either way."""
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    x, y, t, p = make_events(77, 9_000_001, 260, 346)
    ref = oracle.voxel_f32(x, y, t, p, 5, (260, 346))
    pageable = [torch.from_numpy(a) for a in (x, y, t, p)]
    assert not pageable[0].is_pinned()
    out = events_to_voxel_torch(*pageable, 5, sensor_size=(260, 346))
    assert not out.is_cuda
    assert_close_to_max(out.numpy(), ref, 1e-5, "pageable")
    pinned = [a.pin_memory() for a in pageable]
    out2 = events_to_voxel_torch(*pinned, 5, sensor_size=(260, 346))
    assert_close_to_max(out2.numpy(), ref, 1e-5, "pinned")
    out3 = events_to_voxel_torch(*pageable, 5, sensor_size=(260, 346))          # bounce buffers reused across calls
    assert_close_to_max(out3.numpy(), ref, 1e-5, "pageable again")
    # the storage layout (int16, int16, float64, uint8 -- what h5py returns) through the same bounce slots: three chunks
    from event_utils_b200.representations.voxel_grid import events_to_voxel_packed
    xi, yi = x.astype(np.int16), y.astype(np.int16)
    t64 = t.astype(np.float64) * 0.2 + 1.7e9
    pb = (p > 0).astype(np.uint8)
    rel = (t64 - t64[0]).astype(np.float32)
    refp = oracle.voxel_f32(xi, yi, rel, np.where(pb > 0, 1.0, -1.0).astype(np.float32), 5, (260, 346), t0=0.0, dt=rel[-1])
    packed = [torch.from_numpy(a) for a in (xi, yi, t64, pb)]
    assert_close_to_max(events_to_voxel_packed(*packed, 5, sensor_size=(260, 346)).numpy(), refp, 1e-5, "packed pageable")
    assert_close_to_max(events_to_voxel_packed(*(a.pin_memory() for a in packed), 5, sensor_size=(260, 346)).numpy(), refp, 1e-5,
                        "packed pinned")
    assert_close_to_max(events_to_voxel_torch(*pageable, 5, sensor_size=(260, 346)).numpy(), ref, 1e-5, "f32 after packed")


def test_data_loader_arrays(oracle):
    """The arrays DynamicH5Dataset.get_events hands over (hdf5_dataset.py:18-23): int16 coordinates,
    float64 absolute timestamps, float64 +-1 polarities, all numpy."""
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch, events_to_voxel_torch
    x, y, t, p = make_events(41, 200000, 180, 240)
    xi, yi = x.astype(np.int16), y.astype(np.int16)
    t64 = t.astype(np.float64) * 0.25 + 1.6e9        # absolute stamps: not representable in float32
    p64 = p.astype(np.float64)
    rel = (t64 - t64[0]).astype(np.float32)
    ref = oracle.voxel_f32(xi, yi, rel, p, 5, (180, 240), t0=0.0, dt=rel[-1])
    out = events_to_voxel_torch(xi, yi, t64, p64, 5, sensor_size=(180, 240))
    assert not out.is_cuda and out.dtype == torch.float32
    assert_close_to_max(out.numpy(), ref, 1e-5)
    vp, vn = events_to_neg_pos_voxel_torch(xi, yi, t64, p64, 5, sensor_size=(180, 240))
    assert_close_to_max((vp - vn).numpy(), ref, 1e-5)
    # the single all-zero event of BaseVoxelDataset.preprocess_events (base_dataset.py:218-223): dt == 0 -> NaN
    z = np.zeros(1)
    out = events_to_voxel_torch(z, z, z, z, 5, sensor_size=(180, 240))
    assert torch.isnan(out[:, 0, 0]).all() and int(torch.isnan(out).sum()) == 5


def test_packed_storage_layout(oracle):
    """int16 / int16 / float64 / bool arrays as stored on disk -> the same grid as the cast float32 path."""
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_packed
    x, y, t, p = make_events(51, 1_300_001, 260, 346)
    xi, yi = x.astype(np.int16), y.astype(np.int16)
    t64 = t.astype(np.float64) * 0.2 + 1.7e9
    pb = p > 0
    rel = (t64 - t64[0]).astype(np.float32)
    ref = oracle.voxel_f32(xi, yi, rel, np.where(pb, 1.0, -1.0).astype(np.float32), 5, (260, 346), t0=0.0, dt=rel[-1])
    for variant in VARIANTS:
        eu.config.variant = variant
        out = events_to_voxel_packed(xi, yi, t64, pb, 5, sensor_size=(260, 346))
        assert not out.is_cuda
        assert_close_to_max(out.numpy(), ref, 1e-5, variant)
    # contiguous host tensors in the storage dtypes take the chunked H2D pipeline
    out = events_to_voxel_packed(*(torch.from_numpy(a) for a in (xi, yi, t64, pb)), 5, sensor_size=(260, 346))
    assert_close_to_max(out.numpy(), ref, 1e-5)
    out = events_to_voxel_packed(*dev(xi, yi, t64, pb.astype(np.uint8)), 5, sensor_size=(260, 346))
    assert out.is_cuda
    assert_close_to_max(out.cpu().numpy(), ref, 1e-5)
    with pytest.raises(IndexError):
        events_to_voxel_packed(np.int16([400, 1]), np.int16([1, 1]), np.float64([0, 1]), np.uint8([1, 0]), 3, sensor_size=(260, 346))


def test_numpy_flavour_and_negpos(oracle):
    from event_utils_b200.representations.voxel_grid import (events_to_neg_pos_voxel_torch, events_to_voxel)
    g = golden("voxel_numpy")
    for tag in "ab":
        out = events_to_voxel(g[tag + "_x"], g[tag + "_y"], g[tag + "_t"], g[tag + "_p"], int(g[tag + "_B"]),
                              sensor_size=tuple(int(v) for v in g[tag + "_HW"]))
        assert out.dtype == np.float64
        assert_close_to_max(out, g[tag + "_out"], 1e-5, tag)
    with pytest.raises(TypeError):
        events_to_voxel(np.float64([1.0]), np.float64([1.0]), np.float64([0.0]), np.float64([1.0]), 2)
    with pytest.raises(ValueError):
        events_to_voxel(np.int64([-1, 2]), np.int64([1, 1]), np.float64([0.0, 1.0]), np.float64([1.0, 1.0]), 2)
    g = golden("voxel_torch")
    vp, vn = events_to_neg_pos_voxel_torch(*dev(g["np_x"], g["np_y"], g["np_t"], g["np_p"]), 4, sensor_size=(24, 32))
    assert_close_to_max(vp.cpu().numpy(), g["np_pos"], 1e-5)
    assert_close_to_max(vn.cpu().numpy(), g["np_neg"], 1e-5)


def test_negpos_fused_large(oracle):
    """One-pass neg/pos split against two oracle voxel builds, both kernel variants, incl. p == 0."""
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch
    x, y, t, p = make_events(31, 1500003, 120, 160)
    p[::7] = 0.0
    rp = oracle.voxel_f32(x, y, t, (p > 0).astype(np.float32), 5, (120, 160))
    rn = oracle.voxel_f32(x, y, t, (p <= 0).astype(np.float32), 5, (120, 160))
    for variant in VARIANTS:
        eu.config.variant = variant
        vp, vn = events_to_neg_pos_voxel_torch(*dev(x, y, t, p), 5, sensor_size=(120, 160))
        assert_close_to_max(vp.cpu().numpy(), rp, 1e-5, variant)
        assert_close_to_max(vn.cpu().numpy(), rn, 1e-5, variant)
    vp, vn = events_to_neg_pos_voxel_torch(*(torch.from_numpy(a) for a in (x, y, t, p)), 5, sensor_size=(120, 160))
    assert not vp.is_cuda
    assert_close_to_max(vn.numpy(), rn, 1e-5)


def test_windows_helpers(oracle):
    from event_utils_b200.representations.voxel_grid import (events_to_voxel_timesync_torch, voxel_grids_fixed_n_torch)
    x, y, t, p = make_events(12, 50000, 60, 80)
    X, Y, T, P = dev(x, y, t, p)
    grids = voxel_grids_fixed_n_torch(X, Y, T, P, 5, 12000, sensor_size=(60, 80))
    assert len(grids) == 4
    for k, gk in enumerate(grids):
        sl = slice(12000 * k, 12000 * (k + 1))
        assert_close_to_max(gk.cpu().numpy(), oracle.voxel_f32(x[sl], y[sl], t[sl], p[sl], 5, (60, 80)), 1e-5)
    from event_utils_b200.representations.voxel_grid import voxel_grids_fixed_t_torch
    gt = voxel_grids_fixed_t_torch(X, Y, T, P, 4, 0.021, sensor_size=(60, 80))
    t_starts = np.arange(t[0], t[-1] - 0.021, 0.021)
    assert len(gt) == len(t_starts) and len(gt) >= 3
    for k, t0 in enumerate(t_starts):
        i0, i1 = np.searchsorted(t, t0), np.searchsorted(t, t0 + 0.021)
        assert_close_to_max(gt[k].cpu().numpy(), oracle.voxel_f32(x[i0:i1], y[i0:i1], t[i0:i1], p[i0:i1], 4, (60, 80)), 1e-5)
    # non-contiguous / CPU inputs take the per-window fallback and agree
    gl = voxel_grids_fixed_n_torch(*(torch.from_numpy(a) for a in (x, y, t, p)), 5, 12000, sensor_size=(60, 80))
    assert len(gl) == 4 and not gl[0].is_cuda
    assert_close_to_max(gl[2].numpy(), grids[2].cpu().numpy(), 1e-5)
    v = events_to_voxel_timesync_torch(X, Y, T, P, 3, 0.02, 0.06, sensor_size=(60, 80))
    i0, i1 = np.searchsorted(t, 0.02), np.searchsorted(t, 0.06)
    assert_close_to_max(v.cpu().numpy(), oracle.voxel_f32(x[i0:i1], y[i0:i1], t[i0:i1], p[i0:i1], 3, (60, 80)), 1e-5)


def test_c_abi_direct_trilinear_and_windows(oracle):
    """Straight through the C ABI: explicit t0/dt (sharded callers), the trilinear extension and
    the batched-window entry point."""
    from event_utils_b200 import _lib
    L = _lib.lib()
    x, y, t, p = make_events(13, 120000, 48, 64, pol="real")
    X, Y, T, P = dev(x, y, t, p)
    B, H, W = 5, 48, 64
    out = torch.empty((B, H, W), device="cuda")
    ws = torch.empty(L.evk_voxel_workspace_bytes(B, H, W, 0), dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    # a shard [30000, 90000) of the stream with the GLOBAL t0/dt
    t0, dt = float(t[0]), float(np.float32(t[-1]) - np.float32(t[0]))
    sl = slice(30000, 90000)
    for variant in (_lib.VARIANT_GLOBAL_RED, _lib.VARIANT_VECTOR_RED):
        _lib.check(L.evk_voxel_f32(X[sl].data_ptr(), Y[sl].data_ptr(), T[sl].data_ptr(), P[sl].data_ptr(), 60000,
                                   t0, dt, B, H, W, variant, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                   oob.data_ptr(), None))
        torch.cuda.synchronize()
        assert_close_to_max(out.cpu().numpy(), oracle.voxel_f32(x[sl], y[sl], t[sl], p[sl], B, (H, W), t0=t0, dt=dt), 1e-5)
    assert int(oob.item()) == 0
    # trilinear: oracle = per-bin bilinear image with the bin weight folded into the polarity
    tn = (t - np.float32(t0)) / np.float32(dt) * np.float32(B - 1)
    ref = np.stack([oracle.image_torch_f32(x, y, p * np.maximum(0, 1 - np.abs(tn - b)).astype(np.float32),
                                           sensor_size=(H, W), interpolation='bilinear') for b in range(B)])
    out3 = torch.empty((B, H + 1, W + 1), device="cuda")
    ws3 = torch.empty(L.evk_voxel_workspace_bytes(B, H + 1, W + 1, _lib.BILINEAR), dtype=torch.uint8, device="cuda")
    for variant in (_lib.VARIANT_GLOBAL_RED, _lib.VARIANT_VECTOR_RED):
        _lib.check(L.evk_voxel_f32(X.data_ptr(), Y.data_ptr(), T.data_ptr(), P.data_ptr(), x.shape[0], t0, dt, B,
                                   H + 1, W + 1, variant | _lib.BILINEAR | _lib.CLIP, out3.data_ptr(), ws3.data_ptr(),
                                   ws3.numel(), oob.data_ptr(), None))
        torch.cuda.synchronize()
        assert_close_to_max(out3.cpu().numpy(), ref, 1e-5)
    # windows
    offs = np.array([0, 10000, 10000, 45000, 120000], dtype=np.int64)
    outw = torch.empty((4, B, H, W), device="cuda")
    _lib.check(L.evk_voxel_windows_f32(X.data_ptr(), Y.data_ptr(), T.data_ptr(), P.data_ptr(),
                                       torch.from_numpy(offs).cuda().data_ptr(), 4, 120000, B, H, W, 0,
                                       outw.data_ptr(), oob.data_ptr(), None))
    torch.cuda.synchronize()
    for w in range(4):
        a, b = offs[w], offs[w + 1]
        refw = oracle.voxel_f32(x[a:b], y[a:b], t[a:b], p[a:b], B, (H, W)) if b > a else np.zeros((B, H, W), np.float32)
        assert_close_to_max(outw[w].cpu().numpy(), refw, 1e-5, "window %d" % w)


@pytest.mark.parametrize("variant", VARIANTS)
def test_full_size_properties(variant):
    """BASELINE config 2 size (50 M events, 5x480x640): size-independent properties only."""
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    eu.config.variant = variant
    n = 50_000_000
    gen = torch.Generator(device="cuda").manual_seed(2024)
    x = torch.rand(n, device="cuda", generator=gen) * 639
    y = torch.rand(n, device="cuda", generator=gen) * 479
    t = torch.sort(torch.rand(n, device="cuda", generator=gen)).values
    p = (torch.randint(0, 2, (n,), device="cuda", generator=gen) * 2 - 1).float()
    v = events_to_voxel_torch(x, y, t, p, 5, sensor_size=(480, 640))
    total = float(v.double().sum())
    assert abs(total - float(p.double().sum())) <= 2.0        # temporal weights sum to 1 per event
    # |p| = 1: the L1 mass of an all-positive run equals N
    v1 = events_to_voxel_torch(x, y, t, torch.ones_like(p), 5, sensor_size=(480, 640))
    assert abs(float(v1.double().sum()) - n) <= 1e-6 * n
    assert float(v1.min()) >= 0.0
    # linearity: V(p) = V(p>0) - V(p<=0), and additivity over a split of the stream (global t0/dt)
    vpos = events_to_voxel_torch(x, y, t, (p > 0).float(), 5, sensor_size=(480, 640))
    assert_close_to_max((2 * vpos - v1).cpu().numpy(), v.cpu().numpy(), 1e-5)
    # idempotence / determinism of the count-like grid up to fp addition order
    v2 = events_to_voxel_torch(x, y, t, p, 5, sensor_size=(480, 640))
    assert_close_to_max(v2.cpu().numpy(), v.cpu().numpy(), 1e-5)


def test_sharded_stream_single_process(oracle):
    """parallel.ShardedVoxelStream without a process group: buffers recycle correctly and every build
    equals the direct call (the NCCL leg is exercised by bench.py --gpus N and the gloo test)."""
    from event_utils_b200.parallel import ShardedVoxelStream, events_to_voxel_sharded
    x, y, t, p = make_events(91, 300000, 90, 120)
    X, Y, T, P = dev(x, y, t, p)
    pipe = ShardedVoxelStream(5, (90, 120), X.device, depth=2)
    outs = []
    for k in range(5):
        sl = slice(k * 50000, (k + 2) * 50000)
        t0, dt = float(t[sl][0]), float(np.float32(t[sl][-1]) - np.float32(t[sl][0]))
        grid, done = pipe.submit(X[sl], Y[sl], T[sl], P[sl], t0, dt)
        done.synchronize()
        outs.append((grid.clone(), sl, t0, dt))
    pipe.drain()
    for g, sl, t0, dt in outs:
        assert_close_to_max(g.cpu().numpy(), oracle.voxel_f32(x[sl], y[sl], t[sl], p[sl], 5, (90, 120), t0=t0, dt=dt), 1e-5)
    full = events_to_voxel_sharded(X, Y, T, P, 5, (90, 120))
    assert_close_to_max(full.cpu().numpy(), oracle.voxel_f32(x, y, t, p, 5, (90, 120)), 1e-5)



def test_loader_window_tables_one_launch(oracle):
    """every window of a loader table in one launch == get_voxel_grid per window (base_dataset.py:433-455),
    combined and neg/pos channels, overlapping windows, an empty window, host and device inputs"""
    from event_utils_b200.data_loaders import windows as Wn
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch, events_to_voxel_torch
    x, y, t, p = make_events(31, 60000, 40, 52)
    xd, yd, td, pd = dev(x, y, t, p)
    tables = [Wn.k_event_indices(len(x), 7000, 2000)[:-1], Wn.timeblock_indices(t, 0.013, 0.0),
              np.array([[0, 10], [10, 10], [10, 60000], [59999, 60000]])]
    for table in tables:
        for combined in (True, False):
            got = Wn.voxelize_event_windows(xd, yd, td, pd, table, 5, (40, 52), combined_voxel_channels=combined)
            assert got.shape == (len(table), 5 if combined else 10, 40, 52)
            for w, (i0, i1) in enumerate(table):
                if i1 == i0:
                    assert float(got[w].abs().sum()) == 0.0
                    continue
                sl = slice(int(i0), int(i1))
                if combined:
                    want = oracle.voxel_f32(x[sl], y[sl], t[sl], p[sl], 5, (40, 52))
                    single = events_to_voxel_torch(xd[sl], yd[sl], td[sl], pd[sl], 5, sensor_size=(40, 52))
                else:
                    want = np.concatenate((oracle.voxel_f32(x[sl], y[sl], t[sl], (p[sl] > 0).astype(np.float32), 5, (40, 52)),
                                           oracle.voxel_f32(x[sl], y[sl], t[sl], (p[sl] <= 0).astype(np.float32), 5, (40, 52))))
                    single = torch.cat(events_to_neg_pos_voxel_torch(xd[sl], yd[sl], td[sl], pd[sl], 5, sensor_size=(40, 52)), 0)
                if np.isnan(want).any():
                    assert np.array_equal(np.isnan(want), np.isnan(got[w].cpu().numpy()))
                    assert np.array_equal(np.isnan(want), np.isnan(single.cpu().numpy()))
                    continue
                assert_close_to_max(got[w].cpu().numpy(), want, 1e-5)
                assert_close_to_max(got[w].cpu().numpy(), single.cpu().numpy(), 1e-5)
    host = Wn.voxelize_event_windows(*(torch.from_numpy(a) for a in (x, y, t, p)), tables[0], 5, (40, 52))
    assert torch.equal(host, Wn.voxelize_event_windows(xd, yd, td, pd, tables[0], 5, (40, 52))) or \
        float((host - Wn.voxelize_event_windows(xd, yd, td, pd, tables[0], 5, (40, 52))).abs().max()) < 1e-4
    with pytest.raises(Exception):
        Wn.voxelize_event_windows(xd, yd, td, pd, [[0, 60001]], 5, (40, 52))


def test_fold_allreduce_kernel_on_one_device(oracle):
    """evk_voxel_fold_allreduce_f32 with the peers emulated on one GPU: world 1 == the ordinary fold; world 3 (three shards, three workspaces, three grids, one call per emulated rank) == the whole
    stream, and all grids are bit-identical."""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, H, W = 5, 37, 53
    x, y, t, p = make_events(41, 200000, H, W)
    xd, yd, td, pd = dev(x, y, t, p)
    t0, dt = float(t[0]), float(np.float32(t[-1]) - np.float32(t[0]))
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    wsb = L.evk_voxel_workspace_bytes(B, H, W, 0)

    def scatter(lo, hi, ws):
        _lib.check(L.evk_voxel_f32(xd[lo:hi].data_ptr(), yd[lo:hi].data_ptr(), td[lo:hi].data_ptr(), pd[lo:hi].data_ptr(), hi - lo, t0, dt,
                                   B, H, W, _lib.NO_FOLD, None, ws.data_ptr(), ws.numel(), oob.data_ptr(), None))

    ref = torch.empty((B, H, W), device="cuda")
    wsr = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_voxel_f32(xd.data_ptr(), yd.data_ptr(), td.data_ptr(), pd.data_ptr(), len(x), t0, dt, B, H, W, _lib.VARIANT_VECTOR_RED,
                               ref.data_ptr(), wsr.data_ptr(), wsr.numel(), oob.data_ptr(), None))
    even = lambda w: [(200000 * r // w, 200000 * (r + 1) // w) for r in range(w)]   # noqa: E731  (2, 4, 8: unrolled kernels)
    for bounds in ([(0, 200000)], [(0, 70000), (70000, 70000), (70000, 200000)], even(2), even(4), even(8)):
        world = len(bounds)
        wss = [torch.empty(wsb, dtype=torch.uint8, device="cuda") for _ in range(world)]
        outs = [torch.full((B, H, W), float("nan"), device="cuda") for _ in range(world)]
        for (lo, hi), ws in zip(bounds, wss):
            scatter(lo, hi, ws)
        pw = (ctypes.c_void_p * world)(*[w.data_ptr() for w in wss])
        po = (ctypes.c_void_p * world)(*[o.data_ptr() for o in outs])
        for r in range(world):
            _lib.check(L.evk_voxel_fold_allreduce_f32(pw, po, world, r, B, H, W, 0, None))
        torch.cuda.synchronize()
        for o in outs[1:]:
            assert torch.equal(o, outs[0])
        assert_close_to_max(outs[0].cpu().numpy(), ref.cpu().numpy(), 2e-6)   # two runs of float atomics: order differs
        assert_close_to_max(outs[0].cpu().numpy(), oracle.voxel_f32(x, y, t, p, B, (H, W)), 1e-5)
    assert int(oob) == 0
    assert L.evk_voxel_fold_allreduce_f32(pw, po, 17, 0, B, H, W, 0, None) == -1
    assert L.evk_voxel_f32(xd.data_ptr(), yd.data_ptr(), td.data_ptr(), pd.data_ptr(), len(x), t0, dt, B, H, W, _lib.NO_FOLD,
                           None, None, 0, oob.data_ptr(), None) != 0          # NO_FOLD needs the workspace


def _peer_worker(rank, world, port, out_dir):
    import os
    import sys
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from event_utils_b200.parallel import PeerReducedVoxel, events_to_voxel_sharded, shard_bounds
    B, H, W = 5, 60, 80
    x, y, t, p = make_events(43, 300001, H, W)
    lo, hi = shard_bounds(len(x), world, rank)
    sh = [torch.from_numpy(a[lo:hi]).cuda() for a in (x, y, t, p)]
    t0, dt = float(t[0]), float(np.float32(t[-1]) - np.float32(t[0]))
    fused = PeerReducedVoxel(B, (H, W), torch.device("cuda", rank))
    for _ in range(3):                                    # the buffers are reused call after call
        grid = fused(*sh, t0, dt).clone()
    nccl = events_to_voxel_sharded(*sh, B, (H, W), t0=t0, dt=dt)
    nvls = PeerReducedVoxel(B, (H, W), torch.device("cuda", rank), multicast=True)     # through the switch where available
    grid_mc = nvls(*sh, t0, dt).clone() if nvls.multicast else grid
    np.save(os.path.join(out_dir, "peer%d.npy" % rank), np.stack((grid.cpu().numpy(), nccl.cpu().numpy(), grid_mc.cpu().numpy())))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_peer_reduced_voxel_two_gpus(oracle, tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    mp.spawn(_peer_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    a, b = np.load(tmp_path / "peer0.npy"), np.load(tmp_path / "peer1.npy")
    assert np.array_equal(a[0], b[0])                     # bit-identical on both ranks
    x, y, t, p = make_events(43, 300001, 60, 80)
    want = oracle.voxel_f32(x, y, t, p, 5, (60, 80))
    assert_close_to_max(a[0], want, 1e-5)
    assert_close_to_max(a[1], want, 1e-5)
    assert np.array_equal(a[2], b[2])
    assert_close_to_max(a[2], want, 1e-5)


def test_two_threads_two_streams(oracle):
    """scratch buffers are per stream and the host pipeline per thread: concurrent callers do not disturb
    each other (device inputs on side streams, host inputs through the pipeline)"""
    import threading
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    sets = [make_events(70 + k, 1 << 21, 60, 80) for k in range(2)]     # >= 2^20 events: the workspace path
    want = [oracle.voxel_f32(*ev, 5, (60, 80)) for ev in sets]
    errors = []

    def work(k):
        try:
            torch.cuda.set_device(0)
            side = torch.cuda.Stream()
            host = [torch.from_numpy(a) for a in sets[k]]
            with torch.cuda.stream(side):
                on_dev = [a.cuda() for a in host]
                for _ in range(10):
                    got = events_to_voxel_torch(*on_dev, 5, sensor_size=(60, 80))
                    side.synchronize()
                    assert_close_to_max(got.cpu().numpy(), want[k], 1e-5)
                    got_h = events_to_voxel_torch(*host, 5, sensor_size=(60, 80))
                    assert_close_to_max(got_h.numpy(), want[k], 1e-5)
        except Exception as exc:      # surfaced in the main thread
            errors.append(repr(exc))

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
