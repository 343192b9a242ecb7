"""The generators of the planar and camera models' candidates-pass tests, with the f64 references and no GPU: the
candidate sets share no component, GONE keeps no event and PARTIAL 10-90 % of every stream it scores, every event is
safe under every candidate of its window, and the sparse streams put at most one tap on any pixel under every
candidate."""
import numpy as np
import pytest

import candidate_checks as C
import test_gpu_camera_motion as CM
import test_gpu_camera_rotation as CRT
import test_gpu_planar_motion as PM

FAMILIES = {"affine": (PM, ("affine",), PM.cand_warp("affine")), "homography": (PM, ("homography",), PM.cand_warp("homography")),
            "camera_rotation": (CRT, (), CRT.cand_warp()), "camera_motion": (CM, (), CM.cand_warp())}


def _warped(warp, stream, lo, hi, prm):
    x, y, d, _, rho, _ = stream
    return warp(x[lo:hi], y[lo:hi], d[lo:hi], rho[lo:hi], prm)


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("batch", [1, 5, 6])
def test_candidate_sets_and_their_streams(family, batch):
    mod, args, warp = FAMILIES[family]
    cand, stream = mod.candidate_case(*args, batch)
    off = stream[-1]
    assert cand.shape[:2] == (batch, 70) and list(np.diff(off)) == mod.CAND_SIZES[batch]
    C.assert_distinct(cand)
    C.assert_distinct(C.with_nan(cand))
    assert np.isnan(C.with_nan(cand)).sum() == 1 and np.isnan(C.with_nan(cand)[0, C.NAN]).sum() == 1
    for b in range(batch):
        lo, hi = off[b], off[b + 1]
        if hi == lo:
            continue
        warped = [_warped(warp, stream, lo, hi, q) for q in cand[b]]
        assert C.safe(warped).all(), (family, b)
        kept = C.kept(warped, mod.H, mod.W)
        assert not kept[C.GONE].any(), (family, b, kept[C.GONE].sum())
        if hi - lo > 1000:
            share = kept[C.PARTIAL].mean()
            assert 0.1 <= share <= 0.9, (family, b, share)
            assert kept[0].mean() > 0.25, (family, b, kept[0].mean())
            if family == "homography":
                assert np.isnan(warped[C.PARTIAL][0]).any(), b           # events past the horizon


@pytest.mark.parametrize("family", ["affine", "homography", "camera_rotation"])
@pytest.mark.parametrize("M", [2, 3, 4])
def test_segmentation_sets_and_their_streams(family, M):
    mod, args, warp = FAMILIES[family]
    cand, stream = mod.segmentation_case(*args, M)
    assert cand.shape[:3] == (6, M, 37)
    C.assert_distinct(cand)
    off = stream[-1]
    for b in range(6):
        if off[b + 1] > off[b]:
            assert C.safe([_warped(warp, stream, off[b], off[b + 1], q) for q in cand[b].reshape(-1, cand.shape[-1])]).all()


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_sparse_streams_have_one_tap_per_pixel(family):
    mod, args, _ = FAMILIES[family]
    sparse = np.array(mod.SPARSE[args[0]] if args else mod.SPARSE)
    C.assert_distinct(sparse[None])
    case = mod.sparse_case(*args)
    off = case[-1]
    n = off[1]
    assert n > 500, n
    if family == "camera_motion":
        x, y, d, _, rho = (a[:n] for a in case[:5])
        warp = CM.cand_warp(CM.CAMERA)
    else:
        x, y, d = (a[:n] for a in case[:3])
        rho = None
        warp = PM.cand_warp(args[0], (120.0, 90.0)) if args else CRT.cand_warp(CRT.CAMERA)
    warped = [warp(x, y, d, rho, q) for q in sparse]
    assert C.kept(warped, 180, 240).all() and C.safe(warped).all()
    for xw, yw in warped:
        assert C.taps_per_pixel(xw, yw, 180, 240) == 1
