"""No-GPU checks of the image-space tail's reference (tests/tail_reference.py) and of the blur-sigma rule of the C ABI.

1. The kernel's blur rules (reflect_idx, make_taps, mix_coeffs of csrc/evk_cmax.cu), transcribed, equal scipy's blur for
   every canvas and sigma of the GPU sweep (tests/test_gpu_image_tails.py), radii far beyond the canvas and n = 1 included.
2. The bounds are tight enough: an emulated f32 blur with the right rules stays inside them, and one with a wrong radius,
   a wrong boundary mode, a halo one pixel off or swapped channel-mix coefficients is rejected.
3. Every entry point that takes a blur sigma rejects NaN (EVK_E_ARG) and a sigma whose radius exceeds 64 (EVK_E_UNSUPPORTED)
   before it makes any CUDA call."""
import ctypes
import os
import re

import numpy as np
import pytest

import tail_reference as T
from flow_objective_reference import blur_matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the GPU sweep: sigma -> radius 0, 0, 1, 4, 8, 8, 9, 12, 32, 64, 64
SIGMAS = [0.0, 0.1, 0.125, 1.0, 1.875, 2.1249, 2.125, 3.0, 7.9, 15.875, 16.0]
# legacy sensor sizes (Hs, Ws) -> canvas (Hs + 1, Ws + 1); the blur entry also takes (Hs, Ws) itself as an image shape
LEGACY = [(1, 1), (1, 300), (300, 1), (6, 30), (7, 31), (8, 32), (180, 240), (255, 255)]
BATCHED = [(2, 2), (3, 70), (8, 31), (45, 60), (130, 7)]
LENGTHS = sorted({n for hw in LEGACY for n in hw} | {n + 1 for hw in LEGACY for n in hw} | {n + 1 for hw in BATCHED for n in hw})


def test_sweep_radii():
    assert [T.radius(s) for s in SIGMAS] == [0, 0, 1, 4, 8, 8, 9, 12, 32, 64, 64]
    assert T.radius(2.1249) == T.FUSED_MAX_R and T.radius(2.125) == T.FUSED_MAX_R + 1


@pytest.mark.parametrize("sigma", SIGMAS)
def test_transcribed_rules_equal_scipy(sigma):
    """reflect_idx + make_taps along one axis == scipy's gaussian_filter1d (mode reflect, truncate 4) for every length
    of the sweep (1 .. 301: r >> n and n = 1 included), and mix_coeffs == scipy's blur of the 2-stack"""
    for n in LENGTHS:
        err = np.abs(T.kernel_blur_matrix(n, sigma) - blur_matrix(n, sigma)).max()
        assert err <= 1e-15, (n, sigma, err)
    if sigma > 0:
        a, b = T.mix_coeffs(T.taps(sigma))
        ra, rb = T.mix64(sigma)
        assert abs(a - ra) <= 1e-15 and abs(b - rb) <= 1e-15, (sigma, a, b, ra, rb)
        assert abs(a + b - 1.0) <= 1e-15


def test_reflect_rule_known_answers():
    # d c b a | a b c d | d c b a
    assert [T.reflect_idx(i, 4) for i in range(-5, 10)] == [3, 3, 2, 1, 0, 0, 1, 2, 3, 3, 2, 1, 0, 0, 1]
    assert [T.reflect_idx(i, 1) for i in (-70, -1, 0, 1, 70)] == [0] * 5
    assert [T.reflect_idx(i, 2) for i in range(-4, 6)] == [0, 1, 1, 0, 0, 1, 1, 0, 0, 1]


def _image(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


SHAPES = [(hs + 1, ws + 1) for hs, ws in LEGACY[:6]] + [(1, 300), (300, 1), (3, 71), (46, 61)]


@pytest.mark.parametrize("sigma", SIGMAS)
def test_emulated_kernel_blur_is_within_the_bound(sigma):
    for k, shape in enumerate(SHAPES):
        I = _image(shape, k)
        G = T.emulate_blur32(I, sigma)
        err = np.abs(G - T.blur64(I, sigma))
        assert (err <= T.blur_bound(I, sigma)).all(), (shape, sigma, err.max())


def _rejected(I, sigma, **mutation):
    G = T.emulate_blur32(I, sigma, **mutation)
    return (np.abs(G - T.blur64(I, sigma)) > T.blur_bound(I, sigma)).any()


# a mutation of the taps moves a cell by about (the weight it adds or drops) x |I|; below sigma = 1 the weight at r + 1
# (exp(-(r+1)^2 / 2 sigma^2) <= e^-32 at sigma 0.125) is under f32 rounding, so no test can see it, and with the reflect
# rule's n = 1 special case the boundary modes agree on a length-1 axis.  On an axis much shorter than the radius the
# reflection folds the taps at +-(r + 1) onto pixels that already carry nearly the same weight, so a radius change is
# only visible where some axis is longer than the radius.
@pytest.mark.parametrize("sigma", [s for s in SIGMAS if s >= 1.0])
def test_bounds_reject_a_wrong_radius_mode_or_halo(sigma):
    r = T.radius(sigma)
    for k, shape in enumerate(s for s in SHAPES if min(s) >= 2):
        I = _image(shape, 100 + k)
        mutations = [{"mode": "mirror"}, {"mode": "nearest"}, {"shift": 1}, {"shift": -1}]
        if max(shape) > r + 1:
            mutations += [{"dr": -1}, {"dr": 1}]
        for mutation in mutations:
            assert _rejected(I, sigma, **mutation), (shape, sigma, mutation)


def test_bounds_reject_a_halo_shift_at_every_radius():
    for sigma in [s for s in SIGMAS if s > 0]:
        for k, shape in enumerate(SHAPES):
            I = _image(shape, 200 + k)
            assert _rejected(I, sigma, shift=1), (shape, sigma)


OBJECTIVES = [("variance", 0.0), ("sos", 0.0), ("soe", 0.0), ("moa", 0.0), ("isoa", 0.1), ("sosa", 0.3)]


def _emulated_tail(I, D, sigma, name, param, swap=False):
    """the legacy tail's f and mixed gradient computed from the emulated f32 blur (mix coefficients swapped on request)"""
    G = T.emulate_blur32(I, sigma).astype(np.float64)
    I64, D64 = I.astype(np.float64), D.astype(np.float64)
    P = I.size
    w = {"variance": 2 * (G - I64.mean()), "sos": 2 * I64, "soe": np.exp(G), "isoa": (G > np.float32(param)).astype(np.float64),
         "sosa": -param * np.exp(-param * G)}[name]
    c = 1.0 / P if name in ("variance", "sos", "soe") else 1.0
    if name == "variance":
        u = [-c * (w * D64[k]).sum() for k in range(2)]
    else:
        u = [-c * (T.blur64(w, sigma) * D64[k]).sum() for k in range(2)]
    a, b = T.mix_coeffs(T.taps(sigma)) if sigma > 0 else (1.0, 0.0)
    if swap:
        a, b = b, a
    return a * u[0] + b * u[1], b * u[0] + a * u[1]


@pytest.mark.parametrize("name,param", [o for o in OBJECTIVES if o[0] != "moa"])
def test_gradient_bounds_hold_and_reject_swapped_mix_coefficients(name, param):
    """The emulated tail's mixed gradient is inside the bound; with a and b swapped it is not.  A swap only changes the
    gradient by (a - b)(u0 - u1), and a - b is the 2-stack blur's response at a quarter cycle, exp(-2 pi^2 sigma^2 / 16):
    1.5e-5 at sigma 3 and under 1e-15 from sigma 4 up, so the swap is checked where a - b >= 0.003 (sigma 1 to 2.125)."""
    rng = np.random.default_rng(7)
    for shape in [(7, 31), (9, 33), (46, 61)]:
        I = (rng.standard_normal(shape) * (0.3 if name in ("soe", "sosa") else 1.0)).astype(np.float32)
        D = np.stack([rng.standard_normal(shape), 3.0 * rng.standard_normal(shape) + 1.0]).astype(np.float32)
        for sigma in [s for s in SIGMAS if s > 0]:
            ref = T.tail(I, D, sigma, name, param)
            g = _emulated_tail(I, D, sigma, name, param)
            for k in range(2):
                want, bound = ref["g%d" % k]
                assert abs(g[k] - want) <= bound, (shape, sigma, k, g[k], want, bound)
            if 1.0 <= sigma <= 2.125:
                gs = _emulated_tail(I, D, sigma, name, param, swap=True)
                assert any(abs(gs[k] - ref["g%d" % k][0]) > ref["g%d" % k][1] for k in range(2)), (shape, sigma)


@pytest.mark.parametrize("name,param", OBJECTIVES)
def test_f_bounds_hold_for_the_emulated_blur_and_reject_a_wrong_radius(name, param):
    rng = np.random.default_rng(11)
    I = (rng.standard_normal((46, 61)) * (0.3 if name in ("soe", "sosa") else 1.0)).astype(np.float32)
    for sigma in SIGMAS:
        ref = T.tail(I, None, sigma, name, param)
        for mutation, must_hold in (({}, True), ({"dr": 1}, False)):
            if not must_hold and sigma < 1.0:
                continue
            G = T.emulate_blur32(I, sigma, **mutation)
            g64 = G.astype(np.float64)
            f = {"variance": -g64.var(), "sos": -(G * G).astype(np.float64).mean(), "soe": -np.exp(g64).mean(),
                 "moa": -g64.max(), "isoa": float((G > np.float32(param)).sum()), "sosa": -np.exp(-param * g64).sum()}[name]
            want, bound = ref["f"]
            if must_hold:
                assert abs(f - want) <= bound, (sigma, f, want, bound)
            elif name in ("variance", "sos"):      # a max, a count or a sum of exponentials of nearly the mean may not move
                assert abs(f - want) > bound, (sigma, mutation, f, want, bound)


# ---- the blur-sigma rule of the C ABI ------------------------------------------------------------------------------------
SIGMA_ENTRIES = ["evk_cmax_linvel_variance_f64", "evk_cmax_linvel_variance_f32", "evk_cmax_linvel_objective_f64",
                 "evk_cmax_linvel_objective_f32", "evk_cmax_linvel_objective_batch_f64", "evk_cmax_warp_objective_f64",
                 "evk_cmax_warp_objective_f32", "evk_cmax_warp_objective_batch_f64", "evk_iwe_objective_f32",
                 "evk_variance_objective_f32", "evk_gaussian_blur_f32", "evk_cmax_peer_tail_f32", "evk_cmax_flow_variance_f32",
                 "evk_cmax_flow_objective_f32", "evk_cmax_flow_objective_grad_f32", "evk_cmax_motion_objective_f32",
                 "evk_cmax_motion_objective_grad_f32", "evk_flow_timestamp_objective_f32", "evk_flow_timestamp_objective_grad_f32"]


def _sigma_prototypes():
    src = open(os.path.join(ROOT, "include", "evk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\bint\s+(evk_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        params = [p.strip() for p in m.group(2).replace("\n", " ").split(",")]
        if "double sigma" in params:
            out[m.group(1)] = params.index("double sigma")
    return out


def test_every_entry_that_takes_a_sigma_is_covered():
    assert sorted(_sigma_prototypes()) == sorted(SIGMA_ENTRIES)


@pytest.mark.parametrize("name", SIGMA_ENTRIES)
def test_bad_sigma_is_rejected_before_any_cuda_call(name):
    """Called with fake, aligned, never dereferenced pointers, an otherwise plausible argument list and a huge workspace:
    a NaN sigma is EVK_E_ARG and a sigma needing a radius over 64 (16.125 -> 65, 1e9, +inf) is EVK_E_UNSUPPORTED, each
    with a message that names the sigma.  Without a GPU here, a call that reached CUDA could not return those codes."""
    from event_utils_b200 import _lib
    L = _lib.load()
    fn = getattr(L, name)
    at = fn.argtypes
    where = _sigma_prototypes()[name]
    fake = ctypes.c_void_p(1 << 20)
    ptrs = (ctypes.c_void_p * 4)(1 << 20, 1 << 20, 1 << 20, 1 << 20)     # host arrays of device pointers (peer tail)
    defaults = {ctypes.c_void_p: fake, ctypes.c_int64: 10, ctypes.c_double: 1.0, ctypes.c_float: 1.0, ctypes.c_int: 4,
                ctypes.c_uint: 0, ctypes.c_size_t: 1 << 40}
    args = [defaults[t] for t in at]
    if name == "evk_cmax_peer_tail_f32":
        args[0], args[1], args[2] = ptrs, ptrs, 1
    assert at[where] is ctypes.c_double
    for sigma, rc in ((float("nan"), -1), (16.125, -5), (1e9, -5), (float("inf"), -5)):
        args[where] = sigma
        assert fn(*args) == rc, (name, sigma)
        msg = L.evk_last_error()
        assert b"blur sigma" in msg and msg.startswith(b"evk_"), (name, sigma, msg)
    # the largest sigma with radius 64 passes the rule (and then fails elsewhere: no GPU, fake pointers) -- not run here
