"""Multi-GPU voxel build and contrast-maximisation evaluation: one process per GPU, events
partitioned across ranks, ONE sum all-reduce of the (B,H,W) grid -- or of the image of warped events
and its two derivative images -- over NCCL / NVLink.

Every output of the hot path is a sum over events (index_put_(accumulate=True), reference
image.py:95), so any partition of the events works.  The only global quantities are the two
scalars voxel_grid.py:133-134 derives from the whole stream (first timestamp, duration): they
are agreed with two scalar all-reduces (MIN / MAX) -- or passed in when known a priori -- and
handed to the kernel as explicit t0 / dt.  With contiguous time shards each rank touches only
about (B-1)/G + 1 bin planes, but the reduce is over the whole grid (6.1 MB at 5x480x640, latency
bound on NVLink), one collective per call.
"""
import torch
import torch.distributed as dist


def bind_to_gpu_numa_node(device_index=None):
    """Pin the calling process to the CPUs of the NUMA node its GPU hangs off (NVML's ideal CPU affinity for the
    device), BEFORE it allocates pinned host buffers: pinned pages are placed on the node of the allocating thread,
    and a rank whose staging buffers sit on the other socket feeds its GPU through the inter-socket link, which caps
    its host-to-device rate well below what the PCIe link could carry.  One process per GPU; returns the CPU set
    it bound to, or None where NVML / sched_setaffinity are not available (nothing is changed then)."""
    import os
    try:
        import pynvml as nv
        nv.nvmlInit()
        idx = torch.cuda.current_device() if device_index is None else int(device_index)
        try:    # honour CUDA_VISIBLE_DEVICES: go through the UUID of the torch device
            handle = nv.nvmlDeviceGetHandleByUUID(("GPU-" + str(torch.cuda.get_device_properties(idx).uuid)).encode())
        except Exception:
            handle = nv.nvmlDeviceGetHandleByIndex(idx)
        ncpu = os.cpu_count() or 1
        words = nv.nvmlDeviceGetCpuAffinity(handle, (ncpu + 63) // 64)
        cpus = {64 * w + b for w, bits in enumerate(words) for b in range(64) if (int(bits) >> b) & 1}
        allowed = os.sched_getaffinity(0)
        cpus = (cpus & allowed) or None
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return sorted(cpus)
    except Exception:
        return None


def shard_bounds(n, world_size, rank):
    """Contiguous shard [lo, hi) of n events for `rank` (sizes differ by at most one)."""
    base, rem = divmod(int(n), int(world_size))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def global_time_span(ts_local, group=None):
    """(t0, dt) of the WHOLE stream from each rank's (possibly empty) time-sorted shard."""
    dev = ts_local.device
    if ts_local.numel():
        lohi = torch.stack((ts_local[0], -ts_local[-1])).to(torch.float32)
    else:
        lohi = torch.tensor([float("inf"), float("inf")], dtype=torch.float32, device=dev)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(lohi, op=dist.ReduceOp.MIN, group=group)
    first, neg_last = lohi.tolist()
    import numpy as np
    t0 = np.float32(first)
    dt = np.float32(-neg_last) - t0      # f32 subtraction, like ts[-1]-ts[0] on f32 tensors
    return float(t0), float(dt)


def _voxel_local_cuda(xs, ys, ts, ps, t0, dt, B, H, W):
    from .representations.voxel_grid import _voxel_device
    if xs.numel() == 0:
        return torch.zeros((B, H, W), dtype=torch.float32, device=xs.device)
    return _voxel_device(xs, ys, ts, ps, t0, dt, B, H, W)


def events_to_voxel_sharded(xs, ys, ts, ps, B, sensor_size=(180, 240), group=None, t0=None, dt=None,
                            compute=None):
    """
    Voxel grid of a stream whose events are spread over the ranks of `group` (each rank passes
    ITS shard: contiguous f32 tensors on its own GPU).  Every rank returns the full (B,H,W) grid.
    @param t0, dt global first timestamp / duration if already known (skips the two scalar reduces)
    @param compute local kernel `(xs,ys,ts,ps,t0,dt,B,H,W) -> tensor`; defaults to the CUDA path
           (tests inject the CPU oracle to exercise the collective logic with gloo)
    """
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if t0 is None or dt is None:
        t0, dt = global_time_span(ts, group)
    compute = compute or _voxel_local_cuda
    grid = compute(xs, ys, ts, ps, t0, dt, int(B), H, W)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(grid, op=dist.ReduceOp.SUM, group=group)
    return grid


def _image_local_cuda(xs, ys, ps, sensor_size, interpolation):
    from .representations.image import events_to_image_torch
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if xs.numel() == 0:
        pad = 1 if interpolation == 'bilinear' else 0
        return torch.zeros((H + pad, W + pad), dtype=torch.float32, device=xs.device)
    return events_to_image_torch(xs, ys, ps, sensor_size=(H, W), interpolation=interpolation, clip_out_of_range=interpolation == 'bilinear')


def events_to_image_sharded(xs, ys, ps, sensor_size=(180, 240), interpolation=None, group=None, compute=None):
    """
    Event image (reference image.py:46-100, events_to_image_torch) of a stream whose events are spread over the ranks of
    `group`: each rank scatters ITS shard (hot-spot streams through the shared-memory table of csrc/evk_hot.cu), ONE sum
    all-reduce of the image joins them.  An image is a plain sum over events, so any partition works and there is no
    global quantity to agree on.  Every rank returns the full image.
    @param compute local kernel `(xs, ys, ps, sensor_size, interpolation) -> tensor` (tests inject the CPU oracle)
    """
    img = (compute or _image_local_cuda)(xs, ys, ps, sensor_size, interpolation)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(img, op=dist.ReduceOp.SUM, group=group)
    return img


class _PeerBarrier:
    """Cross-GPU barrier on a CUDA stream for the fused peer kernels (evk_peer_barrier): `world` 32-bit slots per rank in
    symmetric memory, one tiny kernel per barrier (a launch + one NVLink round trip).  Default: the symmetric-memory handle's
    own barrier; `EVK_PEER_BARRIER=evk` selects evk_peer_barrier (tools/bench_peer_latency.py times the multi-GPU calls with
    either)."""

    def __init__(self, device, group, handle_for_fallback):
        import ctypes
        import os
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        self._lib, self.L = _lib, _lib.lib()
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.fallback = handle_for_fallback if os.environ.get("EVK_PEER_BARRIER", "torch") == "torch" else None
        self.epoch = 0
        if self.fallback is None:
            self.slots = symm.empty(64, dtype=torch.int32, device=device)
            self.slots.zero_()
            h = symm.rendezvous(self.slots, group)
            self.ptrs = (ctypes.c_void_p * self.world)(*[int(a) for a in h.buffer_ptrs])
            torch.cuda.synchronize(device)
            dist.barrier(group)                 # every rank's slots are zero before anybody signals

    def __call__(self, stream_handle, channel=0):
        if self.fallback is not None:
            self.fallback.barrier(channel=channel)
            return
        self.epoch += 1
        self._lib.check(self.L.evk_peer_barrier(self.ptrs, self.world, self.rank, self.epoch, stream_handle))


class ShardedVoxelStream:
    """Back-to-back sharded voxel builds (a data loader voxelising window after window): the sum
    all-reduce of build k runs on a communication stream and overlaps the scatter kernel of build
    k+1, which the NVLink transfer (6 MB) and its launch latency would otherwise serialise with.
    `submit()` returns the grid buffer and the event that marks its all-reduce complete; buffers are
    recycled round-robin (`depth` in flight)."""

    def __init__(self, B, sensor_size, device, group=None, depth=2):
        self.B, self.H, self.W = int(B), int(sensor_size[0]), int(sensor_size[1])
        self.device, self.group = torch.device(device), group
        self.grids = [torch.empty((self.B, self.H, self.W), dtype=torch.float32, device=self.device) for _ in range(depth)]
        self.done = [torch.cuda.Event() for _ in range(depth)]
        self.comm = torch.cuda.Stream(self.device)
        self.k = 0
        self.multi = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1

    def submit(self, xs, ys, ts, ps, t0, dt):
        from . import _lib
        from .representations.voxel_grid import _voxel_device
        i = self.k % len(self.grids)
        self.k += 1
        cur = torch.cuda.current_stream(self.device)
        if self.k > len(self.grids):
            cur.wait_event(self.done[i])            # the buffer's previous all-reduce must have finished
        _voxel_device(xs, ys, ts, ps, t0, dt, self.B, self.H, self.W, out=self.grids[i])
        if self.multi:
            ready = torch.cuda.Event()
            ready.record(cur)
            self.comm.wait_event(ready)
            with torch.cuda.stream(self.comm):
                dist.all_reduce(self.grids[i], op=dist.ReduceOp.SUM, group=self.group)
                self.done[i].record(self.comm)
        else:
            self.done[i].record(cur)
        return self.grids[i], self.done[i]

    def drain(self):
        """Make the current stream wait for every outstanding all-reduce."""
        cur = torch.cuda.current_stream(self.device)
        for ev in self.done[: min(self.k, len(self.done))]:
            cur.wait_event(ev)


class PeerReducedVoxel:
    """Sharded voxel build whose fold and all-reduce are ONE kernel over NVLink peer memory instead of a
    fold kernel followed by an NCCL all-reduce: every rank scatters its shard into a quad workspace that
    lives in symmetric memory (torch.distributed._symmetric_memory: the same allocation mapped into every
    peer), a cross-GPU barrier, then each rank reduces ITS slice of the pixels over all ranks' workspaces
    with 16-byte peer loads, folds the quads into the B bins and stores the result into every rank's grid
    (evk_voxel_fold_allreduce_f32), and a second barrier.  Per GPU that moves (N-1)/N x 9.8 MB in and
    (N-1)/N x 6.1 MB out at 5x480x640 and costs two barriers; every cell is computed once, so all ranks hold
    bit-identical grids (an NCCL ring all-reduce does not promise that).

    One instance = one grid shape.  `depth` buffers are recycled round-robin: with depth >= 2, `submit()`
    runs barrier + reduce kernel + barrier of build k on a communication stream while build k+1 scatters
    (the interface of ShardedVoxelStream); `__call__` is the synchronous single build."""

    def __init__(self, B, sensor_size, device, group=None, depth=1, multicast=False):
        """multicast=True: reduce and fan out through the NVSwitch (NVLS multimem.ld_reduce / multimem.st on the
        buffers' multicast addresses) where the symmetric-memory backend provides them; the per-GPU link traffic
        then stays 9.8 MB / N in + 6.1 MB / N out for any N.  Falls back to the peer-pointer kernel otherwise
        (`self.multicast` says which is in use)."""
        import ctypes
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        self._lib, self.L = _lib, _lib.lib()
        self.B, self.H, self.W = int(B), int(sensor_size[0]), int(sensor_size[1])
        self.device = torch.device(device)
        group = dist.group.WORLD if group is None else group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        ws_bytes = self.L.evk_voxel_workspace_bytes(self.B, self.H, self.W, _lib.VARIANT_VECTOR_RED)   # the quad workspace
        self.bufs = []
        for _ in range(int(depth)):
            ws = symm.empty(ws_bytes, dtype=torch.uint8, device=self.device)
            out = symm.empty((self.B, self.H, self.W), dtype=torch.float32, device=self.device)
            h_ws, h_out = symm.rendezvous(ws, group), symm.rendezvous(out, group)
            buf = dict(ws=ws, out=out, h_ws=h_ws, h_out=h_out,
                       peer_ws=(ctypes.c_void_p * self.world)(*[int(a) for a in h_ws.buffer_ptrs]),
                       peer_out=(ctypes.c_void_p * self.world)(*[int(a) for a in h_out.buffer_ptrs]),
                       done=torch.cuda.Event(), mc_ws=None, mc_out=None)
            if multicast and int(getattr(h_ws, "multicast_ptr", 0) or 0) and int(getattr(h_out, "multicast_ptr", 0) or 0):
                buf["mc_ws"] = (ctypes.c_void_p * self.world)(*([int(h_ws.multicast_ptr)] * self.world))
                buf["mc_out"] = (ctypes.c_void_p * self.world)(*([int(h_out.multicast_ptr)] * self.world))
            self.bufs.append(buf)
        self.multicast = all(b["mc_ws"] is not None for b in self.bufs)
        self.barrier = _PeerBarrier(self.device, group, self.bufs[0]["h_ws"])
        self.oob = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.comm = torch.cuda.Stream(self.device) if depth > 1 else None
        self.k = 0

    def _reduce(self, buf, stream_handle):
        _lib, L = self._lib, self.L
        self.barrier(stream_handle, 0)            # every rank's reductions have landed in its workspace
        if self.multicast:
            _lib.check(L.evk_voxel_fold_allreduce_f32(buf["mc_ws"], buf["mc_out"], self.world, self.rank, self.B, self.H,
                                                      self.W, _lib.PEER_MULTICAST, stream_handle))
        else:
            _lib.check(L.evk_voxel_fold_allreduce_f32(buf["peer_ws"], buf["peer_out"], self.world, self.rank, self.B, self.H,
                                                      self.W, 0, stream_handle))
        self.barrier(stream_handle, 1)            # every rank's slice has been written into every grid

    def submit(self, xs, ys, ts, ps, t0, dt):
        """This rank's shard (contiguous f32 CUDA tensors) and the stream's global (t0, dt).  Returns the
        (B,H,W) grid buffer -- identical on every rank once complete -- and the event that marks it complete.
        Out-of-grid events are counted in `self.oob`."""
        _lib, L = self._lib, self.L
        buf = self.bufs[self.k % len(self.bufs)]
        self.k += 1
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream(self.device)
            if self.k > len(self.bufs):
                cur.wait_event(buf["done"])       # the buffer's previous reduce has finished on every rank
            _lib.check(L.evk_voxel_f32(_lib.ptr(xs), _lib.ptr(ys), _lib.ptr(ts), _lib.ptr(ps), xs.shape[0], t0, dt,
                                       self.B, self.H, self.W, _lib.NO_FOLD, None, _lib.ptr(buf["ws"]), buf["ws"].numel(),
                                       _lib.ptr(self.oob), cur.cuda_stream))
            if self.comm is None:
                self._reduce(buf, cur.cuda_stream)
                buf["done"].record(cur)
            else:
                ready = torch.cuda.Event()
                ready.record(cur)
                self.comm.wait_event(ready)
                with torch.cuda.stream(self.comm):
                    self._reduce(buf, self.comm.cuda_stream)
                    buf["done"].record(self.comm)
        return buf["out"], buf["done"]

    def __call__(self, xs, ys, ts, ps, t0, dt):
        out, done = self.submit(xs, ys, ts, ps, t0, dt)
        torch.cuda.current_stream(self.device).wait_event(done)
        return out

    def drain(self):
        """Make the current stream wait for every outstanding reduce."""
        cur = torch.cuda.current_stream(self.device)
        for buf in self.bufs[: min(self.k, len(self.bufs))]:
            cur.wait_event(buf["done"])


# ---------------------------------------------------------------------------------------------
# contrast maximisation over a sharded stream (SURVEY 8e: partial IWE + derivative images ->
# all-reduce 523 KB -> blur / variance replicated on every rank)
# ---------------------------------------------------------------------------------------------
SENSOR_SIZE = (180, 240)     # the reference's fixed IWE canvas, objectives.py:191-192


def global_last_timestamp(ts_local, group=None):
    """Last timestamp of the WHOLE stream (the reference warps every event to ts[-1],
    objectives.py:186) from each rank's time-sorted shard, as a Python float (f64)."""
    last = ts_local[-1:].to(torch.float64) if ts_local.numel() else torch.full((1,), float("-inf"), dtype=torch.float64,
                                                                               device=ts_local.device)
    last = last.clone()
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(last, op=dist.ReduceOp.MAX, group=group)
    return float(last.item())


def _cmax_images_cuda(params, xs, ys, ts, ps, t_ref, img_size, want_grad, use_polarity):
    """This rank's partial IWE and derivative images, [3][Hs+1][Ws+1] f32, and the number of its
    events that index outside the canvas (evk_cmax_linvel_variance_f64/_f32 with image outputs)."""
    from . import _lib
    L = _lib.lib()
    Hs, Ws = SENSOR_SIZE
    dev = xs.device
    with torch.cuda.device(dev):
        images = torch.zeros((3, Hs + 1, Ws + 1), dtype=torch.float32, device=dev)
        oob = torch.zeros(1, dtype=torch.int64, device=dev)
        n = int(xs.shape[0])
        if n == 0:
            return images, oob
        ws = _lib.scratch("cmax_ws", L.evk_cmax_workspace_bytes(Hs, Ws), dev)
        result = torch.zeros(12, dtype=torch.float64, device=dev)
        flags = (_lib.CMAX_WANT_GRAD if want_grad else 0) | (0 if use_polarity else _lib.CMAX_ABS_POLARITY)
        diwe = images[1:] if want_grad else None
        if ts.dtype == torch.float64:
            x, y, t, p = (a.to(torch.float64).contiguous() for a in (xs, ys, ts, ps))
            _lib.check(L.evk_cmax_linvel_variance_f64(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), n, 1.0,
                                                      float(params[0]), float(params[1]), float(t_ref), int(img_size[0]),
                                                      int(img_size[1]), Hs, Ws, 0.0, flags, _lib.ptr(result), _lib.ptr(images[0]),
                                                      _lib.ptr(diwe), _lib.ptr(ws), ws.numel(), _lib.stream()))
        else:
            x, y, p = (a.to(torch.float32).contiguous() for a in (xs, ys, ps))
            # fast mode: t relative to the reference time, formed in f64 (integer / large absolute stamps), then f32
            t = (ts.to(torch.float64) - float(t_ref)).to(torch.float32).contiguous()
            _lib.check(L.evk_cmax_linvel_variance_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), n, 1.0,
                                                      float(params[0]), float(params[1]), int(img_size[0]), int(img_size[1]),
                                                      Hs, Ws, 0.0, flags, _lib.ptr(result), _lib.ptr(images[0]), _lib.ptr(diwe),
                                                      _lib.ptr(ws), ws.numel(), _lib.stream()))
        oob.copy_(result[4:5])
        return images, oob


class PeerCmax:
    """Sharded contrast-maximisation evaluation whose all-reduce is FUSED into the objective kernel (VERDICT r1 missing #3):
    every rank splats its shard (evk_cmax_linvel_partial_*: the on-chip event pass for large shards) and leaves its planar
    partial images -- IWE and the two derivative images, 3 x 181 x 241 floats -- in symmetric memory; ONE cross-GPU barrier;
    then every rank's tail kernel (evk_cmax_peer_tail_f32) reads all ranks' partial images through NVLink peer pointers,
    sums them in rank order while gathering its tiles, blurs, reduces and writes f, g and the out-of-canvas count into
    pinned host memory.  No NCCL call, no second all-reduce, no .item() between the halves; the partial images are
    double-buffered so that one barrier per evaluation is enough (the barrier of evaluation k+1 orders tail k before the
    partial pass k+2 that reuses its buffer).  (f, g) is bit-identical on all ranks.
    Reference semantics: variance_objective.evaluate_function / evaluate_gradient with linvel_warp, objectives.py:211-264."""

    def __init__(self, device, group=None, sensor_size=(180, 240)):
        import ctypes
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        self._lib, self.L = _lib, _lib.lib()
        self.device = torch.device(device)
        group = dist.group.WORLD if group is None else group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.Hs, self.Ws = int(sensor_size[0]), int(sensor_size[1])
        self.npix = (self.Hs + 1) * (self.Ws + 1)
        words = 3 * self.npix + 4                      # images + the out-of-canvas counter (8 bytes, 8-byte aligned)
        words += words & 1
        self.oob_off = (3 * self.npix + 1) // 2 * 2    # float index of the counter
        self.bufs = []
        for _ in range(2):
            buf = symm.empty(words, dtype=torch.float32, device=self.device)
            h = symm.rendezvous(buf, group)
            ptrs = [int(a) for a in h.buffer_ptrs]
            self.bufs.append(dict(buf=buf, h=h,
                                  img=(ctypes.c_void_p * self.world)(*ptrs),
                                  oob=(ctypes.c_void_p * self.world)(*[a + 4 * self.oob_off for a in ptrs])))
        self.barrier = _PeerBarrier(self.device, group, self.bufs[0]["h"])
        self.ws = torch.empty(self.L.evk_cmax_workspace_bytes(self.Hs, self.Ws), dtype=torch.uint8, device=self.device)
        self.result = torch.zeros(12, dtype=torch.float64).pin_memory()
        self.result_np = self.result.numpy()
        self.k = 0

    def __call__(self, params, xs, ys, ts, ps, img_size, blur_sigma=1.0, t_ref=None, want_grad=True, use_polarity=True,
                 ts_relative=False):
        """This rank's shard (CUDA tensors: f64 = parity mode with absolute stamps + t_ref, f32 = fast mode) -> (f, g).
        ts_relative: the f32 stamps are already relative to the stream's last timestamp (made so once, in f64, by the
        caller: an optimiser evaluates the same shard hundreds of times)."""
        _lib, L = self._lib, self.L
        if t_ref is None and not ts_relative:
            t_ref = global_last_timestamp(ts)
        b = self.bufs[self.k & 1]
        self.k += 1
        flags = (_lib.CMAX_WANT_GRAD if want_grad else 0) | (0 if use_polarity else _lib.CMAX_ABS_POLARITY)
        n = int(xs.shape[0])
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device)
            img_ptr = b["buf"].data_ptr()
            oob_ptr = img_ptr + 4 * self.oob_off
            if ts.dtype == torch.float64:
                x, y, t, p = (a.to(torch.float64).contiguous() for a in (xs, ys, ts, ps))
                _lib.check(L.evk_cmax_linvel_partial_f64(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), n, 1.0, float(params[0]),
                                                         float(params[1]), float(t_ref), int(img_size[0]), int(img_size[1]), self.Hs,
                                                         self.Ws, flags, img_ptr, oob_ptr, _lib.ptr(self.ws), self.ws.numel(), st.cuda_stream))
            else:
                x, y, p = (a.to(torch.float32).contiguous() for a in (xs, ys, ps))
                t = (ts if ts_relative else (ts.to(torch.float64) - float(t_ref))).to(torch.float32).contiguous()
                _lib.check(L.evk_cmax_linvel_partial_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), n, 1.0, float(params[0]),
                                                         float(params[1]), int(img_size[0]), int(img_size[1]), self.Hs, self.Ws, flags,
                                                         img_ptr, oob_ptr, _lib.ptr(self.ws), self.ws.numel(), st.cuda_stream))
            self.barrier(st.cuda_stream, 0)            # every rank's partial images are in place
            _lib.check(L.evk_cmax_peer_tail_f32(b["img"], b["oob"], self.world, self.Hs + 1, self.Ws + 1, float(blur_sigma), flags,
                                                self.result.data_ptr(), _lib.ptr(self.ws), self.ws.numel(), st.cuda_stream))
            st.synchronize()
        res = self.result_np.copy()
        if res[4] != 0:
            raise IndexError("%d warped events index outside the IWE canvas" % int(res[4]))
        import numpy as np
        return float(res[0]), np.array([res[1], res[2]])


def _cmax_tail_cuda(images, blur_sigma, want_grad):
    """(f, g) of the reduced images (evk_variance_objective_f32)."""
    from . import _lib
    L = _lib.lib()
    dev = images.device
    Hc, Wc = int(images.shape[1]), int(images.shape[2])
    with torch.cuda.device(dev):
        ws = _lib.scratch("cmax_ws", L.evk_cmax_workspace_bytes(Hc - 1, Wc - 1), dev)
        result = torch.zeros(12, dtype=torch.float64, device=dev)
        _lib.check(L.evk_variance_objective_f32(_lib.ptr(images[0]), _lib.ptr(images[1:]) if want_grad else None, Hc, Wc,
                                                float(blur_sigma), _lib.CMAX_WANT_GRAD if want_grad else 0, _lib.ptr(result),
                                                _lib.ptr(ws), ws.numel(), _lib.stream()))
        res = result.cpu().numpy()
    import numpy as np
    return float(res[0]), np.array([res[1], res[2]])


def cmax_variance_sharded(params, xs, ys, ts, ps, img_size, blur_sigma=1.0, group=None, t_ref=None,
                          want_grad=True, use_polarity=True, compute_images=None, compute_tail=None):
    """
    variance_objective.evaluate_function / evaluate_gradient with linvel_warp (reference
    objectives.py:211-264) for a stream whose events are spread over the ranks of `group`: every
    rank splats ITS shard (tensors on its own GPU; f64 = parity mode, f32 = fast mode) into a
    partial image of warped events and its two derivative images, ONE sum all-reduce of those
    3 x 181 x 241 floats joins them, and every rank evaluates blur + variance (+ gradient) of the
    full images.  Returns (f, g) -- identical on all ranks.
    @param t_ref the stream's last timestamp if known (skips one scalar all-reduce)
    @param compute_images, compute_tail injection points for the gloo tests (CPU oracle)
    """
    if t_ref is None:
        t_ref = global_last_timestamp(ts, group)
    images, oob = (compute_images or _cmax_images_cuda)(params, xs, ys, ts, ps, t_ref, img_size, want_grad, use_polarity)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(images, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(oob, op=dist.ReduceOp.SUM, group=group)
    if int(oob.item()) != 0:
        raise IndexError("%d warped events index outside the IWE canvas" % int(oob.item()))
    return (compute_tail or _cmax_tail_cuda)(images, blur_sigma, want_grad)
