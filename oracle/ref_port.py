"""Library-op port of the reference's CPU paths -- TEST / BASELINE INFRASTRUCTURE ONLY.

The reference itself (pure Python) is not part of this repository, so where no checkout is named by
$EVK_REFERENCE_ROOT the CPU baseline that bench.py reports (`cpu_baseline.kind == "port"`, and the
`--impl reference` arm) times THIS module: the same sequence of numpy / torch / scipy library calls the reference issues, written
from its documented behaviour (SURVEY.md Appendix A), so that its cost profile -- B passes over
the events, one temporary per elementwise op, `index_put_(accumulate=True)` / `np.bincount`
scatter -- is the reference's.  tests/test_ref_port.py checks it against the golden vectors of
the real reference.

  voxel_torch_cpu   events_to_voxel_torch      lib/representations/voxel_grid.py:129-153
  voxel_numpy       events_to_voxel            lib/representations/voxel_grid.py:198-217
  cmax_fg_cpu       variance_objective f + f'  lib/contrast_max/objectives.py:211-264 via
                    get_iwe :184-192, linvel_warp warps.py:52-60, events_to_image_drv image.py:179-217
"""
import numpy as np
import torch


def _scatter_nearest_torch(canvas, ys_long, xs_long, weights):
    canvas.index_put_((ys_long, xs_long), weights, accumulate=True)
    return canvas


def voxel_torch_cpu(xs, ys, ts, ps, B, sensor_size=(180, 240)):
    """f32 torch tensors on the CPU -> (B,H,W) f32.  One full pass (6 elementwise temporaries,
    two integer casts, one accumulate-scatter) per bin, exactly the reference's cost shape."""
    span = ts[-1] - ts[0]
    tau = (ts - ts[0]) / span * (B - 1)
    floor0 = torch.zeros(tau.size())
    planes = []
    for b in range(B):
        tri = torch.max(floor0, 1.0 - torch.abs(tau - b))
        contrib = ps * tri
        plane = (torch.ones(list(sensor_size)) * 0)
        planes.append(_scatter_nearest_torch(plane, ys.long(), xs.long(), contrib))
    return torch.stack(planes)


def voxel_numpy(xs, ys, ts, ps, B, sensor_size=(180, 240)):
    """integer xs/ys, f64 -> (B,H,W) f64 through np.bincount on an (H+1,W+1) canvas."""
    H, W = sensor_size
    span = ts[-1] - ts[0]
    tau = (ts - ts[0]) / span * (B - 1)
    floor0 = np.zeros(tau.shape[0])
    planes = []
    for b in range(B):
        tri = np.maximum(floor0, 1.0 - np.abs(tau - b))
        contrib = ps * tri
        flat = np.ravel_multi_index(np.stack((ys, xs)), (H + 1, W + 1))
        canvas = np.bincount(flat, weights=contrib, minlength=(H + 1) * (W + 1)).reshape(H + 1, W + 1)
        planes.append(canvas[0:H, 0:W])
    return np.stack(planes)


def _iwe_cpu(params, xs, ys, ts, ps, img_size, want_grad):
    # warps.py:52-60
    lag = ts - ts[-1]
    xw = xs - lag * params[0]
    yw = ys - lag * params[1]
    jx = jy = None
    if want_grad:
        jx = np.zeros((2, len(xw)))
        jy = np.zeros((2, len(yw)))
        jx[0, :] = -lag
        jy[1, :] = -lag
    # event_util.py:26-27 + objectives.py:188-190
    keep = np.where(np.logical_or(xw <= 0, xw > img_size[1]), 0.0, 1.0)
    keep *= np.where(np.logical_or(yw <= 0, yw > img_size[0]), 0.0, 1.0)
    xw, yw, pw = xw * keep, yw * keep, ps * keep
    if want_grad:
        jx, jy = jx * keep, jy * keep
    # image.py:179-217 (fixed 181x241 canvas)
    xt, yt, pt = torch.from_numpy(xw).float(), torch.from_numpy(yw).float(), torch.from_numpy(pw).float()
    inside = torch.where(xt >= 240, torch.tensor([0.]), torch.tensor([1.])) * \
        torch.where(yt >= 180, torch.tensor([0.]), torch.tensor([1.]))
    fx, fy = xt.floor(), yt.floor()
    rx, ry = xt - fx, yt - fy
    ix, iy = (fx * inside).long(), (fy * inside).long()
    wgt = pt * inside
    iwe = torch.zeros((181, 241))
    iwe.index_put_((iy, ix), wgt * (1.0 - rx) * (1.0 - ry), accumulate=True)
    iwe.index_put_((iy, ix + 1), wgt * rx * (1.0 - ry), accumulate=True)
    iwe.index_put_((iy + 1, ix), wgt * (1.0 - rx) * ry, accumulate=True)
    iwe.index_put_((iy + 1, ix + 1), wgt * rx * ry, accumulate=True)
    diwe = None
    if want_grad:
        a1 = torch.from_numpy(jx).float() * wgt
        a2 = torch.from_numpy(jy).float() * wgt
        diwe = torch.zeros((2, 181, 241))
        for k in range(2):
            diwe[k].index_put_((iy, ix), a1[k] * (-(1.0 - ry)) + a2[k] * (-(1.0 - rx)), accumulate=True)
            diwe[k].index_put_((iy, ix + 1), a1[k] * (1.0 - ry) + a2[k] * (-rx), accumulate=True)
            diwe[k].index_put_((iy + 1, ix), a1[k] * (-ry) + a2[k] * (1.0 - rx), accumulate=True)
            diwe[k].index_put_((iy + 1, ix + 1), a1[k] * ry + a2[k] * rx, accumulate=True)
        diwe = diwe.numpy()
    return iwe.numpy(), diwe


def cmax_fg_cpu(params, xs, ys, ts, ps, img_size=(180, 240), blur_sigma=1.0):
    """One optimiser 'iteration' of the reference: evaluate_function THEN evaluate_gradient,
    each rebuilding the IWE from the raw f64 events (objectives.py:227, :250)."""
    from scipy.ndimage import gaussian_filter
    iwe, _ = _iwe_cpu(params, xs, ys, ts, ps, img_size, False)
    if blur_sigma > 0:
        iwe = gaussian_filter(iwe, blur_sigma)
    f = -np.var(iwe - np.mean(iwe))
    iwe, diwe = _iwe_cpu(params, xs, ys, ts, ps, img_size, True)
    if blur_sigma > 0:
        diwe = gaussian_filter(diwe, blur_sigma)
    centred = 2.0 * (iwe - np.mean(iwe))
    g = -np.array([np.mean(centred * diwe[k]) for k in range(2)])
    return f, g
