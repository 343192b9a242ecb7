"""Contrast-maximisation objectives -- drop-in for the hot-path part of the reference's
lib/contrast_max/objectives.py: `objective_function` (base class, :10-140), `get_iwe`
(:165-199) and `variance_objective` (:202-264).

The reference rebuilds everything from the raw host arrays for every f and every f' call
(~25 O(N) numpy/torch passes + 4 or 12 scatters).  Here:
  * the event arrays are uploaded to the GPU once and cached (the optimiser hands over the same
    numpy arrays at every iteration, events_cmax.py:341);
  * warp + bounds mask + IWE + derivative images + blur + variance + gradient is ONE fused
    evaluation (csrc/evk_cmax.cu) that returns f and g together;
  * (params -> f, g) is memoised, so scipy's separate f / f' calls at the same point cost one
    launch.
Objects keep the reference's attributes and calling conventions (positional `args=` form,
keyword form, and the precomputed `iwe=` / `d_iwe=` form).
"""
import threading
from abc import ABC, abstractmethod

import numpy as np
import torch

from .. import _lib
from ..representations import _events as E
from ..representations.image import events_to_image_drv, image_to_event_weights
from ..util.event_util import events_bounds_mask

SENSOR_SIZE = (180, 240)  # the reference never forwards sensor_size to events_to_image_drv
                          # (objectives.py:191-192 -> image.py:163): the IWE is always 181x241


# ---------------------------------------------------------------------------------------------
# device-side event cache
# ---------------------------------------------------------------------------------------------
class _DeviceEvents:
    __slots__ = ("key", "x", "y", "t", "p", "n", "t_last", "mode")


_event_cache = []          # most recent first, at most _CACHE_SLOTS entries
_CACHE_SLOTS = 2
event_pass = None          # None: automatic; "onchip": shared-memory IWE (cmax_onchip_kernel); "l2": L2 vector reductions
precision = "f64"          # "f64": parity mode (events kept as f64, 32 B/event)
                           # "f32": fast mode (x, y, t - t_last, p as f32, 16 B/event)


def _fingerprints(arrays):
    """Identity of host arrays for the caches: length, dtype and a 64-bit hash of EVERY byte
    (evk_host_hash64_multi, threaded above 2 MiB).  The reference's objective is a pure
    function of the arrays it is handed (objectives.py:211-236): a device copy or a memoised result may be
    reused only when the arrays are byte-identical to the ones it was made from -- a sampled fingerprint
    would silently return the previous stream's f / g after a partial in-place edit."""
    return tuple((a.shape[0], a.dtype.str, h) for a, h in zip(arrays, _lib.host_hashes(arrays)))


class pinned_events:
    """Explicit opt-in for optimisation loops: `with pinned_events(xs, ys, ts, ps):` uploads the event
    set once and promises that the four arrays are not modified inside the block, so evaluations that are
    handed the SAME array objects skip the per-call content hash (identity = object ids while the block
    keeps them alive).  Outside such a block every call hashes the full arrays."""
    _active = []

    def __init__(self, xs, ys, ts, ps):
        self.arrays = (xs, ys, ts, ps)
        self.ev = None

    def __enter__(self):
        self.ev = _device_events(*self.arrays)
        pinned_events._active.append(self)
        return self

    def __exit__(self, *exc):
        pinned_events._active.remove(self)
        self.ev = None

    @staticmethod
    def lookup(xs, ys, ts, ps):
        for h in reversed(pinned_events._active):
            a = h.arrays
            if a[0] is xs and a[1] is ys and a[2] is ts and a[3] is ps and h.ev is not None and h.ev.mode == precision:
                return h.ev
        return None


def _device_events(xs, ys, ts, ps):
    ev = pinned_events.lookup(xs, ys, ts, ps)
    if ev is not None:
        return ev
    xs, ys, ts, ps = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1)) for a in (xs, ys, ts, ps))
    key = (precision,) + _fingerprints((xs, ys, ts, ps))
    for i, ev in enumerate(_event_cache):
        if ev.key == key:
            if i:
                _event_cache.insert(0, _event_cache.pop(i))
            return ev
    dev = E.compute_device()
    ev = _DeviceEvents()
    ev.key, ev.n, ev.mode = key, xs.shape[0], precision
    ev.t_last = float(ts[-1]) if ts.shape[0] else 0.0
    with torch.cuda.device(dev):
        # numpy arrays are ordinary pageable memory: _lib.upload stages them through pinned bounce buffers (evk_host_upload)
        if precision == "f64":
            ev.x, ev.y, ev.t, ev.p = _lib.upload([torch.from_numpy(a) for a in (xs, ys, ts, ps)], dev)
        else:
            # relative timestamps in f64, then f32
            ev.x, ev.y, ev.t, ev.p = (a.float() for a in _lib.upload([torch.from_numpy(a) for a in (xs, ys, ts - ev.t_last, ps)], dev))
    _event_cache.insert(0, ev)
    del _event_cache[_CACHE_SLOTS:]
    return ev


def clear_cache():
    del _event_cache[:]


_result_bufs = {}


def _result_buffers(dev):
    """Per-device result buffer reused across evaluations: 12 doubles of PINNED HOST memory that the
    last kernel of an evaluation writes straight over PCIe (pinned allocations are device-addressable
    under unified addressing), so reading a result back is one stream synchronise -- no device buffer,
    no D2H copy operation (a fresh torch.zeros + pageable .cpu() per call, or even a pinned mirror + copy_, is a
    noticeable share of a small evaluation).  Returns (tensor, numpy view)."""
    k = (dev, torch.cuda.current_stream(dev).cuda_stream, threading.get_ident())   # per stream AND host thread: reuse is only safe in stream order
    b = _result_bufs.get(k)
    if b is None:
        host = torch.zeros(12, dtype=torch.float64).pin_memory()
        b = (host, host.numpy())
        _result_bufs[k] = b
    return b


class _on_device:
    """`with torch.cuda.device(dev)` only when dev is not already current (the context manager costs
    several microseconds per evaluation)."""
    __slots__ = ("ctx",)

    def __init__(self, dev):
        self.ctx = None if torch.cuda.current_device() == dev.index else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)


def _fused_linvel(params, xs, ys, ts, ps, img_size, blur_sigma, want_grad, use_polarity,
                  first=0, last=None, p_scale=1.0, want_images=False, channel_mix=True,
                  objective=_lib.OBJ_VARIANCE, obj_param=0.0, ev=None):
    """One fused evaluation on events [first:last) of the cached device copy.
    Returns (result[8] as numpy f64, iwe or None, d_iwe or None)."""
    L = _lib.lib()
    ev = _device_events(xs, ys, ts, ps) if ev is None else ev
    n_all = ev.n
    last = n_all if last is None else (last if last >= 0 else n_all + last)
    first = first if first >= 0 else n_all + first
    first, last = max(0, min(first, n_all)), max(0, min(last, n_all))
    n = max(0, last - first)
    if n == 0:
        raise IndexError("index -1 is out of bounds for axis 0 with size 0")
    Hs, Ws = SENSOR_SIZE
    dev = ev.x.device
    with _on_device(dev):
        ws_bytes = L.evk_cmax_workspace_bytes(Hs, Ws)
        ws = _lib.scratch("cmax_ws", ws_bytes, dev)
        result, result_view = _result_buffers(dev)
        iwe = torch.empty((Hs + 1, Ws + 1), dtype=torch.float32, device=dev) if want_images else None
        d_iwe = torch.empty((2, Hs + 1, Ws + 1), dtype=torch.float32, device=dev) if (want_images and want_grad) else None
        flags = (_lib.CMAX_WANT_GRAD if want_grad else 0) | (0 if use_polarity else _lib.CMAX_ABS_POLARITY) \
            | (0 if channel_mix else _lib.CMAX_NO_CHANNEL_MIX) \
            | {None: 0, "onchip": _lib.VARIANT_SMEM_TILE, "l2": _lib.VARIANT_VECTOR_RED}[event_pass]
        sigma = float(blur_sigma) if blur_sigma is not None else 0.0
        # the reference warps to the LAST timestamp of the (possibly sliced) event set (objectives.py:186)
        if ev.mode == "f64":
            t_ref = float(ev.t[last - 1].item()) if last != n_all else ev.t_last
            off = first * 8
            _lib.check(L.evk_cmax_linvel_objective_f64(
                ev.x.data_ptr() + off, ev.y.data_ptr() + off, ev.t.data_ptr() + off, ev.p.data_ptr() + off, n,
                float(p_scale), float(params[0]), float(params[1]), t_ref, int(img_size[0]), int(img_size[1]),
                Hs, Ws, sigma, flags, int(objective), float(obj_param), _lib.ptr(result), _lib.ptr(iwe), _lib.ptr(d_iwe),
                _lib.ptr(ws), ws.numel(), _lib.stream()))
        else:
            if last != n_all:
                raise NotImplementedError("f32 fast mode stores t relative to the last event; "
                                          "slicing the tail (adaptive_lifespan) needs precision='f64'")
            off = first * 4
            _lib.check(L.evk_cmax_linvel_objective_f32(
                ev.x.data_ptr() + off, ev.y.data_ptr() + off, ev.t.data_ptr() + off, ev.p.data_ptr() + off, n,
                float(p_scale), float(params[0]), float(params[1]), int(img_size[0]), int(img_size[1]),
                Hs, Ws, sigma, flags, int(objective), float(obj_param), _lib.ptr(result), _lib.ptr(iwe), _lib.ptr(d_iwe),
                _lib.ptr(ws), ws.numel(), _lib.stream()))
        torch.cuda.current_stream().synchronize()
        res = result_view.copy()
        if res[4] != 0:
            raise IndexError("%d warped events index outside the IWE canvas %s" % (int(res[4]), (Hs + 1, Ws + 1)))
        return res, (iwe.cpu().numpy() if iwe is not None else None), (d_iwe.cpu().numpy() if d_iwe is not None else None)


def _objective_of_images(iwe, d_iwe, blur_sigma, want_grad, objective=_lib.OBJ_VARIANCE, obj_param=0.0):
    """objective (+ gradient) of precomputed images, on the GPU (evk_iwe_objective_f32)."""
    L = _lib.lib()
    dev = E.compute_device()
    iwe = np.ascontiguousarray(iwe, dtype=np.float32)
    with torch.cuda.device(dev):
        a = torch.from_numpy(iwe).to(dev)
        d = torch.from_numpy(np.ascontiguousarray(d_iwe, dtype=np.float32)).to(dev) if d_iwe is not None else None
        ws = _lib.scratch("cmax_ws", L.evk_cmax_workspace_bytes(iwe.shape[0] - 1, iwe.shape[1] - 1), dev)
        result = torch.zeros(12, dtype=torch.float64, device=dev)
        flags = _lib.CMAX_WANT_GRAD if (want_grad and d is not None) else 0
        _lib.check(L.evk_iwe_objective_f32(_lib.ptr(a), _lib.ptr(d), iwe.shape[0], iwe.shape[1], float(blur_sigma), flags,
                                           int(objective), float(obj_param), _lib.ptr(result), _lib.ptr(ws), ws.numel(),
                                           _lib.stream()))
        return result.cpu().numpy()


# ---------------------------------------------------------------------------------------------
# reference API
# ---------------------------------------------------------------------------------------------
class objective_function(ABC):
    """
    Parent class of the contrast-maximisation objectives (reference objectives.py:10-140):
    same constructor arguments, attributes and housekeeping methods.
    """
    def __init__(self, name="template", use_polarity=True,
            has_derivative=True, default_blur=1.0, adaptive_lifespan=False,
            pixel_crossings=5, minimum_events=10000):
        self.name = name
        self.use_polarity = use_polarity
        self.has_derivative = has_derivative
        self.default_blur = default_blur
        self.adaptive_lifespan = adaptive_lifespan
        self.pixel_crossings = pixel_crossings
        self.minimum_events = minimum_events

        self.recompute_lifespan = True
        self.lifespan = 0.5
        self.s_idx = 0
        self.num_events = None
        self._memo = None   # (key, f, g) of the last fused evaluation
        super().__init__()

    @abstractmethod
    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        pass

    @abstractmethod
    def evaluate_gradient(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None, d_iwe=None):
        pass

    def iter_update(self, params, pixel_crossings=None):
        """Optimiser callback (objectives.py:113-127): new lifespan from the current speed."""
        pixel_crossings = self.pixel_crossings if pixel_crossings is None else pixel_crossings
        magnitude = np.linalg.norm(params)
        if magnitude == 0:
            dt = 5
        else:
            dt = pixel_crossings / magnitude
        self.lifespan = dt
        self.recompute_lifespan = True

    def update_lifespan(self, ts):
        """New start index of the events used when adaptive_lifespan is on (objectives.py:129-140)."""
        if self.adaptive_lifespan:
            self.s_idx = np.searchsorted(ts, ts[-1] - self.lifespan)
            self.s_idx = len(ts) - self.minimum_events if len(ts) - self.s_idx < self.minimum_events else self.s_idx
        if self.num_events is None:
            self.num_events = len(ts) - self.s_idx

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            setattr(new, k, None if k == "_memo" else copy.deepcopy(v, memo))
        return new


def get_iwe(params, xs, ys, ts, ps, warpfunc, img_size, compute_gradient=False,
        use_polarity=True, return_events=False, return_per_event_contrast=False):
    """
    Image of warped events (and dIWE/dparams) for a parameter vector; drop-in for
    objectives.py:165-199.  numpy in, numpy float32 (181,241) / (dims,181,241) out.
    @returns tuple: iwe, d_iwe (or None) [, (xs_warped, ys_warped)] [, per-event contrast]
    """
    fused = getattr(warpfunc, "fused_kind", None) == "linvel"
    if fused and not return_events and not return_per_event_contrast:
        _, iwe, d_iwe = _fused_linvel(params, xs, ys, ts, ps, img_size, 0.0, compute_gradient, use_polarity,
                                      want_images=True)
        return (iwe, d_iwe)
    # generic warp objects (and the two debugging outputs): host warp + mask as in the
    # reference, image formation on the GPU
    xs, ys, ts, ps = (np.asarray(a) for a in (xs, ys, ts, ps))
    if not use_polarity:
        ps = np.abs(ps)
    xw, yw, jx, jy = warpfunc.warp(xs, ys, ts, ps, ts[-1], params, compute_grad=compute_gradient)
    mask = events_bounds_mask(xw, yw, 0, img_size[1], 0, img_size[0])
    xw, yw, ps = xw * mask, yw * mask, ps * mask
    if compute_gradient:
        jx, jy = jx * mask, jy * mask
    iwe, iwe_drv = events_to_image_drv(xw, yw, ps, jx, jy, interpolation='bilinear', compute_gradient=compute_gradient)
    returnval = [iwe, iwe_drv]
    if return_events:
        returnval.append((xw, yw))
    if return_per_event_contrast:
        returnval.append(image_to_event_weights(xw, yw, iwe))
    return tuple(returnval)


class variance_objective(objective_function):
    """
    Variance objective (Gallego & Scaramuzza, RAL'17); drop-in for objectives.py:202-264.
        f(params)   = -var( G_sigma * IWE )
        f'(params)_k = -mean( 2 (IWE - mean IWE) * (G_sigma *3d dIWE)_k )
    Bug-compatible with the reference: the gradient uses the UN-blurred IWE and scipy's 3-D blur
    of the (2,H,W) derivative stack mixes its two channels (objectives.py:253).
    """
    def __init__(self, adaptive_lifespan=False, minimum_events=10000):
        super().__init__(name="variance", use_polarity=True, has_derivative=True,
                default_blur=1.0, adaptive_lifespan=adaptive_lifespan, pixel_crossings=5,
                minimum_events=minimum_events)

    # one fused evaluation returns f and g; remember it for the sibling call at the same point
    def _evaluate(self, params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma):
        first, last, scale = 0, None, 1.0
        if self.adaptive_lifespan:
            if self.recompute_lifespan:
                self.update_lifespan(ts)
                self.recompute_lifespan = False
            first, last, scale = int(self.s_idx), -1, 100.0   # xs[s_idx:-1], ps*100 (objectives.py:224-225)
        blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
        fused = getattr(warpfunc, "fused_kind", None) == "linvel"
        ev = _device_events(xs, ys, ts, ps) if fused else None
        # memo only for the fused warp: a generic warp object's result depends on that object's identity and state
        key = (tuple(float(v) for v in params), ev.key, tuple(img_size), float(blur_sigma), first, last, scale,
               self.use_polarity, precision) if fused else None
        if fused and self._memo is not None and self._memo[0] == key:
            return self._memo[1], self._memo[2]
        if fused:
            res, _, _ = _fused_linvel(params, xs, ys, ts, ps, img_size, blur_sigma, True, self.use_polarity,
                                      first=first, last=last, p_scale=scale, ev=ev)
        else:
            sl = slice(first, last)
            iwe, d_iwe = get_iwe(params, xs[sl], ys[sl], ts[sl], ps[sl] * scale, warpfunc, img_size,
                                 use_polarity=self.use_polarity, compute_gradient=True)
            res = _objective_of_images(iwe, d_iwe, blur_sigma, True)
        f, g = float(res[0]), np.array([res[1], res[2]])
        self._memo = (key, f, g) if fused else None
        return f, g

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        """-var(blurred IWE) at `params` (or of a precomputed `iwe`)."""
        if iwe is not None:
            blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
            return float(_objective_of_images(iwe, None, blur_sigma, False)[0])
        f, _ = self._evaluate(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma)
        return f

    def evaluate_gradient(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None, d_iwe=None):
        """Analytic gradient of the objective wrt the warp parameters (np.ndarray[dims])."""
        if iwe is not None and d_iwe is not None:
            blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
            res = _objective_of_images(iwe, d_iwe, blur_sigma, True)
            return np.array([res[1], res[2]])
        _, g = self._evaluate(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma)
        return g.copy()


# ---------------------------------------------------------------------------------------------
# the reference's other objective functions (objectives.py:266-596) on the same fused event pass
# ---------------------------------------------------------------------------------------------
class _fused_objective(objective_function):
    """Shared machinery: one fused GPU evaluation (event pass + image-space tail) per parameter
    point, memoised so that evaluate_function / evaluate_gradient at the same point cost one
    launch.  Subclasses set `_kind` (an EVK_OBJ_* code) and may override `_param()`."""
    _kind = _lib.OBJ_VARIANCE

    def _param(self):
        return 0.0

    def _result(self, params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma, iwe=None, d_iwe=None, want_grad=True):
        blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
        if iwe is not None:
            return _objective_of_images(iwe, d_iwe, blur_sigma, want_grad and d_iwe is not None, self._kind, self._param())
        fused = getattr(warpfunc, "fused_kind", None) == "linvel"
        ev = _device_events(xs, ys, ts, ps) if fused else None
        key = (tuple(float(v) for v in params), ev.key, tuple(img_size), float(blur_sigma), self.use_polarity,
               precision, self._kind, self._param()) if fused else None
        memo = getattr(self, "_memo", None)
        if fused and memo is not None and memo[0] == key:
            return memo[1]
        if fused:
            res, _, _ = _fused_linvel(params, xs, ys, ts, ps, img_size, blur_sigma, self.has_derivative, self.use_polarity,
                                      objective=self._kind, obj_param=self._param(), ev=ev)
        else:
            img, dimg = get_iwe(params, xs, ys, ts, ps, warpfunc, img_size, use_polarity=self.use_polarity,
                                compute_gradient=self.has_derivative)
            res = _objective_of_images(img, dimg, blur_sigma, self.has_derivative, self._kind, self._param())
        self._memo = (key, res) if fused else None
        return res

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        return float(self._result(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma, iwe=iwe, want_grad=False)[0])

    def evaluate_gradient(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None, d_iwe=None):
        if not self.has_derivative:
            return None
        if iwe is not None and d_iwe is None:
            iwe = None
        res = self._result(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma, iwe=iwe, d_iwe=d_iwe)
        return np.array([res[1], res[2]])


class rms_objective(_fused_objective):
    """"Root mean squared" objective (objectives.py:266-306).  The reference computes
    np.linalg.norm(iwe, 2) on the 2-D image, i.e. its SPECTRAL norm (largest singular value), so
    f = -sigma_max(G*IWE)^2 / npix; f'_k = -2 mean(IWE * (G3d * dIWE)_k).  The event pass and the blur
    run in the evk kernels; the singular value is one torch.linalg call on the 181x241 device image."""
    _kind = _lib.OBJ_SOS

    def __init__(self):
        super().__init__(name="rms", use_polarity=True, has_derivative=True, default_blur=1.0)

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
        if iwe is None:
            iwe, _ = get_iwe(params, xs, ys, ts, ps, warpfunc, img_size, use_polarity=self.use_polarity,
                             compute_gradient=False)
        L = _lib.lib()
        dev = E.compute_device()
        with torch.cuda.device(dev):
            a = torch.from_numpy(np.ascontiguousarray(iwe, dtype=np.float32)).to(dev)
            g, tmp = torch.empty_like(a), torch.empty_like(a)
            _lib.check(L.evk_gaussian_blur_f32(_lib.ptr(a), a.shape[0], a.shape[1], float(blur_sigma), _lib.ptr(g),
                                               _lib.ptr(tmp), _lib.stream()))
            norm = float(torch.linalg.matrix_norm(g.double(), 2))
        return -(norm * norm) / (iwe.shape[0] * iwe.shape[1])


class sos_objective(_fused_objective):
    """Sum of squares objective (Stoffregen et al., CVPR'19; objectives.py:308-356): f = -mean((G*IWE)^2).
    The reference's evaluate_gradient calls an undefined `find_lifespan` (objectives.py:345) and raises
    NameError; the formula it would compute, -mean((G3d*dIWE)_k * 2 IWE), is what is returned here."""
    _kind = _lib.OBJ_SOS

    def __init__(self, adaptive_lifespan=False, minimum_events=10000):
        super().__init__(name="sos", use_polarity=True, has_derivative=True, default_blur=1.0,
                         adaptive_lifespan=adaptive_lifespan, pixel_crossings=5, minimum_events=minimum_events)
        self.current_num_events = minimum_events
        self.div = 1


class soe_objective(_fused_objective):
    """Sum of exponentials objective (objectives.py:358-399): f = -mean(exp(G*IWE)), |p| is used."""
    _kind = _lib.OBJ_SOE

    def __init__(self):
        super().__init__(name="soe", use_polarity=False, has_derivative=True, default_blur=2.5)


class moa_objective(_fused_objective):
    """Max of accumulations objective (objectives.py:401-429): f = -max(G*IWE); no analytic derivative."""
    _kind = _lib.OBJ_MOA

    def __init__(self):
        super().__init__(name="moa", use_polarity=False, has_derivative=False, default_blur=3.0)

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        return float(self._result(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma, iwe=iwe, want_grad=False)[0])


class isoa_objective(_fused_objective):
    """Inverse sum of accumulations objective (objectives.py:431-476): f = +#(G*IWE > thresh) (the
    reference does not negate it), f'_k = -sum((G3d*dIWE)_k [G*IWE > thresh])."""
    _kind = _lib.OBJ_ISOA

    def __init__(self, thresh=0.5):
        super().__init__(name="isoa", use_polarity=False, has_derivative=True, default_blur=1.0)
        self.thresh = thresh

    def _param(self):
        return float(self.thresh)


class sosa_objective(_fused_objective):
    """Sum of suppressed accumulations objective (objectives.py:478-522): f = -sum(exp(-p G*IWE))."""
    _kind = _lib.OBJ_SOSA

    def __init__(self, p=3):
        super().__init__(name="sosa", use_polarity=False, has_derivative=True, default_blur=2.0)
        self.p = p

    def _param(self):
        return float(self.p)


class r1_objective(_fused_objective):
    """R1 objective (objectives.py:560-596): SoS and SoSA combined, with the reference's stateful
    `last_sosa` logic kept literally; no analytic derivative."""
    _kind = _lib.OBJ_SOSA

    def __init__(self, p=3):
        super().__init__(name="r1", use_polarity=False, has_derivative=False, default_blur=1.0)
        self.p = p
        self.last_sosa = 0

    def _param(self):
        return float(self.p)

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        res = self._result(params, xs, ys, ts, ps, warpfunc, img_size, blur_sigma, iwe=iwe, want_grad=False)
        sos, sosa = float(res[8]), float(res[9])
        if sosa > self.last_sosa:
            return -sos
        self.last_sosa = sosa
        return -sos * sosa


class zhu_timestamp_objective(objective_function):
    """Squared timestamp images objective (Zhu et al., CVPR'19; objectives.py:524-558):
        f = -( sum((G * T+)^2) + sum((G * T-)^2) )
    with T+ / T- the average-timestamp images of the warped positive / negative events.  The reference's
    evaluate_function calls `events_to_zhu_timestamp_image`, a name that does not exist anywhere in it
    (NameError, SURVEY Appendix B11); the function it evidently means is `events_to_timestamp_image`
    (image.py:219-284, same argument order, same (pos, neg) return), which is what is used here with its
    defaults -- so this class does what the reference's code says once that one name is resolved.  Warp
    and bounds mask stay on the host as written there (:540-543: x, y, t AND p are multiplied by the mask);
    timestamp images, blur and the two sums run on the GPU."""
    def __init__(self):
        super().__init__(name="zhu", use_polarity=True, has_derivative=False, default_blur=2.0)

    def evaluate_function(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None):
        from ..representations.image import _timestamp_images
        if iwe is not None:
            raise NameError("name 'posimg' is not defined")      # the reference's iwe= branch never defines its images
        xs, ys, ts, ps = (np.asarray(a, dtype=np.float64) for a in (xs, ys, ts, ps))
        xw, yw, _, _ = warpfunc.warp(xs, ys, ts, ps, ts[-1], params, compute_grad=False)
        mask = events_bounds_mask(xw, yw, 0, img_size[1], 0, img_size[0])
        xw, yw, tm, pm = xw * mask, yw * mask, ts * mask, ps * mask
        blur_sigma = self.default_blur if blur_sigma is None else blur_sigma
        L = _lib.lib()
        dev = E.compute_device()
        with torch.cuda.device(dev):
            # events_to_timestamp_image (image.py:241-261): stamps relative to the first, in f64, then f32
            rel = tm - tm[0]
            x, y, p = (torch.from_numpy(np.ascontiguousarray(a)).to(dev).float() for a in (xw, yw, pm))
            t = torch.from_numpy(rel).to(dev).float()
            pos, neg = _timestamp_images(x, y, t, p, 0.0, float(np.float32(rel[-1])), SENSOR_SIZE, True, 'bilinear', True, False)
            total = 0.0
            for img in (pos, neg):
                if blur_sigma > 0:
                    g, tmp = torch.empty_like(img), torch.empty_like(img)
                    _lib.check(L.evk_gaussian_blur_f32(_lib.ptr(img), img.shape[0], img.shape[1], float(blur_sigma), _lib.ptr(g),
                                                       _lib.ptr(tmp), _lib.stream()))
                    img = g
                total += float((img * img).sum())                  # np.sum of an f32 image: f32 pairwise sum
        return -total

    def evaluate_gradient(self, params=None, xs=None, ys=None, ts=None, ps=None,
            warpfunc=None, img_size=None, blur_sigma=None, showimg=False, iwe=None, d_iwe=None):
        """No derivative known (objectives.py:553-558)."""
        return None


def evaluate_candidates(objective, params_list, xs, ys, ts, ps, warpfunc, img_size, blur_sigma=None, want_grad=False):
    """Objective (and gradient) at MANY parameter points with one pass over the events per 32
    candidates (evk_cmax_linvel_objective_batch_f64): what grid_search_initial needs
    (events_cmax.py:300-302 evaluates 25 points per level, one full evaluation each).
    @returns (f[K], g[K,2] or None)"""
    params_list = [tuple(float(v) for v in prm) for prm in params_list]
    kind = getattr(objective, "_kind", _lib.OBJ_VARIANCE)
    prm_fn = getattr(objective, "_param", None)
    obj_param = float(prm_fn()) if prm_fn is not None else 0.0
    sigma = objective.default_blur if blur_sigma is None else blur_sigma
    fused = getattr(warpfunc, "fused_kind", None) == "linvel" and precision == "f64" \
        and not getattr(objective, "adaptive_lifespan", False) and type(objective).evaluate_function in (
            _fused_objective.evaluate_function, variance_objective.evaluate_function)
    if not fused:
        f = np.array([objective.evaluate_function(prm, xs, ys, ts, ps, warpfunc, img_size, blur_sigma) for prm in params_list])
        g = np.array([objective.evaluate_gradient(prm, xs, ys, ts, ps, warpfunc, img_size, blur_sigma)
                      for prm in params_list]) if want_grad else None
        return f, g
    L = _lib.lib()
    ev = _device_events(xs, ys, ts, ps)
    Hs, Ws = SENSOR_SIZE
    dev = ev.x.device
    K = len(params_list)
    out = np.zeros((K, 12))
    with torch.cuda.device(dev):
        ws = _lib.scratch("cmax_ws", L.evk_cmax_workspace_bytes(Hs, Ws), dev)
        flags = (_lib.CMAX_WANT_GRAD if want_grad else 0) | (0 if objective.use_polarity else _lib.CMAX_ABS_POLARITY)
        for lo in range(0, K, 32):
            chunk = np.ascontiguousarray(np.array(params_list[lo:lo + 32], dtype=np.float64).reshape(-1, 2))
            res = torch.zeros((chunk.shape[0], 12), dtype=torch.float64, device=dev)
            _lib.check(L.evk_cmax_linvel_objective_batch_f64(
                ev.x.data_ptr(), ev.y.data_ptr(), ev.t.data_ptr(), ev.p.data_ptr(), ev.n, 1.0,
                chunk.ctypes.data, chunk.shape[0], ev.t_last, int(img_size[0]), int(img_size[1]), Hs, Ws, float(sigma), flags,
                int(kind), obj_param, _lib.ptr(res), _lib.ptr(ws), ws.numel(), _lib.stream()))
            out[lo:lo + chunk.shape[0]] = res.cpu().numpy()
    if out[:, 4].any():
        raise IndexError("warped events index outside the IWE canvas")
    return out[:, 0].copy(), (out[:, 1:3].copy() if want_grad else None)
