/*
 * evk.h -- C ABI of libevk.so: H100 (sm_90a) kernels for the event_utils hot path.
 *
 * The reference (TimoStoff/event_utils) is pure Python and has NO FFI of its own; its
 * "operator API" is a set of module-level Python functions (SURVEY.md section 8b).  Each entry
 * point below is what a ctypes/cffi binding for one of those functions binds to; the reference
 * call site it replaces is cited as file:line (paths relative to the reference tree).
 * INTEGRATION.md shows the ctypes stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every function returns 0 on success, a negative EVK_E_* code on failure; it never throws
 *     across the ABI.  evk_last_error() returns a thread-local human-readable message.
 *   - unless the name says `_host`, all data pointers are caller-owned DEVICE pointers and all
 *     work is enqueued on the caller's stream (a cudaStream_t passed as void*); nothing
 *     synchronises.  No torch types anywhere.
 *   - `oob` (may be NULL) is a device counter the kernels increment once per event whose index
 *     falls outside the output (the reference raises IndexError for those, image.py:96-99);
 *     such events are never written.  The caller zeroes and reads it.
 *   - outputs are fully overwritten unless EVK_ACCUMULATE is set.
 */
#ifndef EVK_H_
#define EVK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define EVK_VERSION 100 /* 0.1.0 */

/* error codes */
#define EVK_OK 0
#define EVK_E_ARG (-1)       /* bad argument (null pointer, negative size, ...) */
#define EVK_E_CUDA (-2)      /* a CUDA runtime call failed, see evk_last_error() */
#define EVK_E_WORKSPACE (-3) /* workspace too small */
#define EVK_E_DEVICE (-4)    /* not an sm_90 device */
#define EVK_E_UNSUPPORTED (-5)

/* flags shared by the scatter entry points */
#define EVK_ACCUMULATE 0x1u   /* add into `out` instead of overwriting it */
#define EVK_BILINEAR 0x2u     /* spatial 4-tap bilinear splat instead of nearest (truncate) */
#define EVK_CLIP 0x4u         /* events_to_image_torch(clip_out_of_range=True) semantics */
#define EVK_AUTO_SPAN 0x200000u    /* voxel: ignore the t0/dt arguments, take t[0] and t[n-1]-t[0] on the device */
#define EVK_WINDOW_PAIRS 0x100000u /* evk_voxel_windows_f32: offsets are (start,end) pairs, 2*n_windows entries */
#define EVK_NO_FOLD 0x800000u /* evk_voxel_f32: leave the sums in the quad workspace (out may be NULL); evk_voxel_fold_allreduce_f32 finishes */
#define EVK_PEER_MULTICAST 0x1000000u /* evk_voxel_fold_allreduce_f32: entry 0 of both pointer arrays is an NVLS multicast address */
#define EVK_WINDOW_NEGPOS 0x400000u /* evk_voxel_windows_f32: out is [n_windows][2][B][H][W], the [p>0] / [p<=0] split per window */
#define EVK_NEGPOS_TRUTHY 0x8u /* neg/pos split on numpy truthiness (p != 0) instead of p > 0 */
#define EVK_WINDOW_OVERLAP 0x2000000u /* evk_voxel_grad_f32: windows may share events; their per-event gradients are added */
#define EVK_EVENTS_AOS 0x4000000u /* evk_voxel_grad_f32: x is one 16-byte aligned (N,4) [x,y,t,p] array; y, t, p are ignored */
/* kernel variant selection, bits 8..11 (0 = pick automatically) */
#define EVK_VARIANT_SHIFT 8
#define EVK_VARIANT_MASK (0xFu << EVK_VARIANT_SHIFT)
#define EVK_VARIANT_AUTO (0u << EVK_VARIANT_SHIFT)
#define EVK_VARIANT_GLOBAL_RED (1u << EVK_VARIANT_SHIFT) /* one scalar red.global.add.f32 per tap */
#define EVK_VARIANT_VECTOR_RED (2u << EVK_VARIANT_SHIFT) /* one red.global.add.v4.f32 per tap pair, quad-layout workspace */
#define EVK_VARIANT_SMEM_TILE (3u << EVK_VARIANT_SHIFT)  /* the shared-memory form of the entry point: voxel / image = vector or scalar reductions behind a per-CTA
                                                          * fixed-point write-combining table (forced on; AUTO probes for contention); cmax = the whole image of
                                                          * warped events in the CTA's shared memory, flushed by TMA bulk reductions (cmax_onchip_kernel) */
#define EVK_VARIANT_WARP_AGG (4u << EVK_VARIANT_SHIFT)   /* warp-aggregated (match.any) global reds, for hot-spot streams */
#define EVK_VARIANT_ROUTED (5u << EVK_VARIANT_SHIFT)     /* voxel: retired, the same as EVK_VARIANT_AUTO (DESIGN.md section 4); the value stays for binary compatibility */

#define EVK_TS_REVERSE 0x80u  /* timestamp images: timestamp_reverse=True (image.py:318-319) */
#define EVK_TS_RAW 0x1000u    /* timestamp images: normalize_timestamps=False (image.py:261): weights = t as given */

/* cmax flags */
#define EVK_CMAX_WANT_GRAD 0x10u    /* also produce the analytic gradient */
#define EVK_CMAX_ABS_POLARITY 0x20u /* use_polarity=False: p <- |p| (objectives.py:184-185) */
#define EVK_CMAX_NO_CHANNEL_MIX 0x40u /* do NOT reproduce the 3-D blur channel mixing (objectives.py:253) */

int evk_version(void);
const char *evk_last_error(void);
/* 0 if the current device is compute capability 9.0 (the library is built for sm_90a only), EVK_E_DEVICE otherwise */
int evk_device_check(void);

/* ---------------------------------------------------------------------------------------------
 * Measurement hooks (bench.py).  With profiling enabled every DOMINANT kernel launch of the
 * scatter entry points (voxel / image scatter, cmax scatter) is bracketed by a CUDA event pair
 * recorded on the launching stream, and every kernel launch of the library is counted.
 * evk_prof_collect() synchronises those events, returns the summed device time of the bracketed
 * launches in *ms, their number in *timed and the total number of kernel launches in *launches,
 * and resets the counters.
 * --------------------------------------------------------------------------------------------- */
int evk_prof_enable(int on);
int evk_prof_collect(double *ms, long long *timed, long long *launches);

/* ---------------------------------------------------------------------------------------------
 * Voxel grid.  Replaces events_to_voxel_torch, lib/representations/voxel_grid.py:114-153
 * (per-bin loop :136-151 -> events_to_image_torch image.py:88-95 -> index_put_).
 *   tau = ((t - t0) / dt) * (B-1)   (f32, this order);  V[b, trunc(y), trunc(x)] += p*max(0,1-|tau-b|)
 * t0, dt are explicit so that a sharded caller can pass the GLOBAL values (voxel_grid.py:133-134
 * derives them from ts[0], ts[-1]).  x,y,t,p: n floats each (SoA), any 4-byte alignment.
 * out: B*H*W floats, layout [B][H][W].
 * With EVK_BILINEAR the spatial part is a 4-tap bilinear splat on the same (H,W) grid
 * (trilinear voxel; an extension, not a reference function).
 * workspace: evk_voxel_workspace_bytes() bytes (may be 0/NULL for the GLOBAL_RED variant).
 * --------------------------------------------------------------------------------------------- */
size_t evk_voxel_workspace_bytes(int B, int H, int W, unsigned flags);
int evk_voxel_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                  float t0, float dt, int B, int H, int W, unsigned flags, float *out,
                  void *workspace, size_t workspace_bytes, unsigned long long *oob, void *stream);

/* Positive and negative events into separate grids in ONE pass.  Replaces
 * events_to_neg_pos_voxel_torch, lib/representations/voxel_grid.py:155-182 (two full
 * events_to_voxel_torch calls with weights [p>0] and [p<=0], :172-175); with EVK_NEGPOS_TRUTHY the
 * numpy flavour's split np.where(ps,1,0) / np.where(ps,0,1) (:234-235).
 * out_pos_neg: 2*B*H*W floats, [0] = positive grid, [1] = negative grid.
 * workspace: 2 * evk_voxel_workspace_bytes(B,H,W,flags) bytes. */
int evk_voxel_negpos_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                         float t0, float dt, int B, int H, int W, unsigned flags, float *out_pos_neg,
                         void *workspace, size_t workspace_bytes, unsigned long long *oob,
                         void *stream);

/* Same, events given as one interleaved (N,4) [x,y,t,p] f32 array (the data-loader layout,
 * lib/data_loaders/base_dataset.py:306,510); ev must be 16-byte aligned. */
int evk_voxel_aos_f32(const float *ev, int64_t n, float t0, float dt, int B, int H, int W,
                      unsigned flags, float *out, void *workspace, size_t workspace_bytes,
                      unsigned long long *oob, void *stream);

/* Same, events in the reference's STORAGE layout (row f4): int16 x, int16 y, float64 t, bool/uint8 p as
 * the HDF5 and memmap formats hold them (lib/data_formats/event_packagers.py:90-93,
 * h5_to_memmap.py:115-117), polarity mapped p*2-1 like the loaders do (hdf5_dataset.py:22,
 * memmap_dataset.py:24).  Timestamps are made relative to t_first in float64, then cast to float32;
 * dt = (float)(t_last - t_first).  13 B/event instead of 16 and no host-side casts. */
int evk_voxel_packed_f32(const int16_t *x, const int16_t *y, const double *t, const uint8_t *p, int64_t n,
                         double t_first, double t_last, int B, int H, int W, unsigned flags, float *out,
                         void *workspace, size_t workspace_bytes, unsigned long long *oob, void *stream);

/* Multi-GPU finish of a sharded voxel build (no reference counterpart: the reference is single-process;
 * SURVEY 8e): after every rank has run evk_voxel_f32(..., EVK_NO_FOLD) on its shard into a workspace that
 * its peers can address (CUDA IPC / symmetric memory over NVLink), and a cross-GPU barrier, each rank calls
 * this once: it reduces ITS slice of the pixels over all ranks' workspaces, folds the temporal quads into
 * the B bins and writes the result into every rank's [B][H][W] grid -- fold and all-reduce in one kernel
 * over peer memory.  A second cross-GPU barrier must follow before the grids are read or the workspaces
 * reused.  peer_workspaces / peer_outs: HOST arrays of `world` device pointers, index = rank.
 * With EVK_PEER_MULTICAST entry 0 of each array is the buffer's NVLS multicast address instead (the
 * other entries are ignored): the NVSwitch sums the quads (multimem.ld_reduce) and fans the result out
 * (multimem.st), so the per-GPU link traffic no longer grows with the number of ranks. */
int evk_voxel_fold_allreduce_f32(const void *const *peer_workspaces, float *const *peer_outs, int world,
                                 int rank, int B, int H, int W, unsigned flags, void *stream);

/* Batched windows (voxel_grids_fixed_n_torch, voxel_grid.py:37-57; BaseVoxelDataset windows,
 * base_dataset.py:322-367): window w covers events [offsets[w], offsets[w+1]) and writes
 * out[w] ([n_windows][B][H][W]); t0/dt per window are taken from the window's first / last
 * timestamp exactly as voxel_grid.py:133-134 does.  offsets: n_windows+1 int64 on the device.
 * With EVK_WINDOW_PAIRS offsets holds 2*n_windows entries, (start,end) per window (windows may then
 * overlap or leave gaps, as events_to_voxel_timesync_torch's do, voxel_grid.py:105-106).
 * With EVK_WINDOW_NEGPOS out is [n_windows][2][B][H][W]: per window the two grids of
 * events_to_neg_pos_voxel_torch (voxel_grid.py:155-182), what BaseVoxelDataset.get_voxel_grid builds
 * with combined_voxel_channels=False (base_dataset.py:449-453).
 * n_events_hint: total number of events covered (0 = unknown), used only to size the launch. */
int evk_voxel_windows_f32(const float *x, const float *y, const float *t, const float *p,
                          const int64_t *offsets, int n_windows, int64_t n_events_hint, int B, int H,
                          int W, unsigned flags, float *out, unsigned long long *oob, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Event image.  Replaces events_to_image_torch, lib/representations/image.py:46-100 and
 * interpolate_to_image, image.py:102-115.
 *   nearest : img[trunc(y)*m, trunc(x)*m] += p           (m = [x<clipx][y<clipy] with EVK_CLIP;
 *             NOTE the weight is not masked, image.py:94-95)
 *   bilinear: 4-tap splat of p*m at floor(x)*m, floor(y)*m with the unmasked fractions
 * Himg, Wimg are the CANVAS sizes (sensor+1 when bilinear and padding, image.py:64-67); the
 * caller derives clipx/clipy as image.py:73-74 does.  `fill` is the background (`default`).
 * --------------------------------------------------------------------------------------------- */
size_t evk_image_workspace_bytes(int Himg, int Wimg, unsigned flags);
int evk_image_f32(const float *x, const float *y, const float *p, int64_t n, int Himg, int Wimg,
                  float clipx, float clipy, unsigned flags, float fill, float *out,
                  void *workspace, size_t workspace_bytes, unsigned long long *oob, void *stream);

/* Average-timestamp images of the positive / negative events.  Replaces
 * events_to_timestamp_image_torch, lib/representations/image.py:286-353 (and the numpy flavour
 * :219-284 after its casts).  t_first / t_last are ts[0] / ts[-1]; Himg, Wimg the canvas
 * (sensor+1 with padding); clipx/clipy as image.py:311-312.  out_pos / out_neg: Himg*Wimg floats.
 * workspace: evk_timestamp_image_workspace_bytes() bytes, 16-byte aligned. */
size_t evk_timestamp_image_workspace_bytes(int Himg, int Wimg);
int evk_timestamp_image_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                            float t_first, float t_last, int Himg, int Wimg, float clipx, float clipy,
                            unsigned flags, float *out_pos, float *out_neg, void *workspace,
                            size_t workspace_bytes, unsigned long long *oob, void *stream);
/* Same, and also writes the count images the division uses (image.py:333-351: one plus the bilinear
 * count, a zero replaced by one) into cnt_pos / cnt_neg (Himg*Wimg floats each), which the backward
 * evk_timestamp_image_grad_f32 needs.  out_pos / out_neg are bit-identical to evk_timestamp_image_f32's. */
int evk_timestamp_image_counts_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                                   float t_first, float t_last, int Himg, int Wimg, float clipx, float clipy,
                                   unsigned flags, float *out_pos, float *out_neg, float *cnt_pos, float *cnt_neg,
                                   void *workspace, size_t workspace_bytes, unsigned long long *oob, void *stream);

/* Integer-exact event-count image (nearest, weight +1 per event): out is u32 [Himg][Wimg].
 * The bit-exact form of events_to_image(_torch) for ps == 1 (image.py:37-38, :95). */
int evk_count_u32(const float *x, const float *y, int64_t n, int Himg, int Wimg, float clipx,
                  float clipy, unsigned flags, unsigned int *out, unsigned long long *oob,
                  void *stream);

/* ---------------------------------------------------------------------------------------------
 * The reference's lower-level splat / gather helpers, for callers that use them directly.
 *   evk_splat_idx_f32       interpolate_to_image, lib/representations/image.py:102-115
 *                           (in place on img [H][W]; px,py int64; dx,dy,w f32)
 *   evk_splat_drv_idx_f32   interpolate_to_derivative_img, image.py:117-136
 *                           (in place on dimg [K][H][W]; w1,w2 are [K][n])
 *   evk_image_drv_f32       events_to_image_drv, image.py:162-217 after its f64->f32 casts
 *                           (:179-183): x,y,p f32, Jacobians jx,jy [K][n] f32 (K may be 0),
 *                           writes img [Himg][Wimg] and dimg [K][Himg][Wimg]
 *   evk_gather_bilinear_f64 image_to_event_weights, image.py:138-160 (f64, img [H][W] f64)
 * --------------------------------------------------------------------------------------------- */
int evk_splat_idx_f32(const int64_t *px, const int64_t *py, const float *dx, const float *dy,
                      const float *w, int64_t n, int H, int W, float *img, unsigned long long *oob,
                      void *stream);
int evk_splat_drv_idx_f32(const int64_t *px, const int64_t *py, const float *dx, const float *dy,
                          const float *w1, const float *w2, int K, int64_t n, int H, int W,
                          float *dimg, unsigned long long *oob, void *stream);
int evk_image_drv_f32(const float *x, const float *y, const float *p, const float *jx, const float *jy,
                      int K, int64_t n, int Himg, int Wimg, float clipx, float clipy, unsigned flags,
                      float *img, float *dimg, unsigned long long *oob, void *stream);
int evk_gather_bilinear_f64(const double *x, const double *y, int64_t n, const double *img, int H,
                            int W, double *out, unsigned long long *oob, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Dense-flow warp.  Replaces warp_events_flow_torch, lib/transforms/optic_flow.py:5-46
 * (F.grid_sample bilinear, align_corners=True, zero padding, :37-44).
 * flow: [2][H][W] f32.  xw/yw: n floats.  x' = x + u(x,y)*(t-t0), y' = y + v(x,y)*(t-t0).
 * workspace (optional, evk_warp_flow_workspace_bytes(), 16-byte aligned): lets the kernel re-lay the
 * flow out as {u,v} pairs so that the two taps of an image row are one 16-byte load.
 * --------------------------------------------------------------------------------------------- */
size_t evk_warp_flow_workspace_bytes(int H, int W);
int evk_warp_flow_f32(const float *x, const float *y, const float *t, int64_t n, const float *flow,
                      int H, int W, float t0, float *xw, float *yw, void *workspace,
                      size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Backward passes.  The reference's torch functions are plain torch ops that autograd runs through
 * (events_to_image_torch image.py:46-100 with interpolate_to_image :102-115, events_to_timestamp_image_torch
 * image.py:286-353, warp_events_flow_torch optic_flow.py:5-46); these entry points give the same gradients
 * for the forward entry points above, one pass over the events each.  Arguments that name the forward's
 * inputs take the values the forward was called with.  Per-event gradient outputs are n floats and may be
 * NULL (not written).  floor() has zero derivative, so gradients are one-sided at integer coordinates.
 *
 *   evk_image_grad_f32   gradient of evk_image_f32 (flags: EVK_BILINEAR, EVK_CLIP) given grad_img
 *                        [Himg][Wimg].  Bilinear: grad_x, grad_y through the fractions x - floor(x),
 *                        y - floor(y) (unmasked, as in the forward), grad_p = mask * the gathered taps.
 *                        Nearest: grad_p = grad_img[trunc(y)*m][trunc(x)*m] (clipped events read [0][0],
 *                        negative indices wrap); grad_x / grad_y are not written (the reference's .long()
 *                        cuts them off).  Events outside the canvas get 0.
 *   evk_timestamp_image_grad_f32
 *                        gradient of evk_timestamp_image_counts_f32 (flags EVK_CLIP, EVK_TS_REVERSE; not
 *                        EVK_TS_RAW) given grad_pos / grad_neg, the outputs and the count images.  Writes
 *                        grad_x, grad_y (through the sum and the count image) and grad_t = g_tn * dtn/dt
 *                        (+-1/D, D = t_last - t_first + 1e-6); sums (2 doubles on the device, may be NULL)
 *                        receives sum(g_tn) and sum(g_tn * tn), from which the caller adds the t_first /
 *                        t_last terms: forward (S1 - S0)/D to t_first and -S1/D to t_last; reverse S1/D to
 *                        t_first and (S0 - S1)/D to t_last.  Polarity gets no gradient.
 *                        workspace: evk_timestamp_image_grad_workspace_bytes() bytes, 16-byte aligned.
 *   evk_warp_flow_grad_f32
 *                        gradient of evk_warp_flow_f32 given grad_xw / grad_yw: grad_x, grad_y (1 + dt * the
 *                        flow's derivative at the sample), grad_t = g_x u + g_y v, *sum_grad_t (one double on
 *                        the device, may be NULL) = sum of grad_t (t0's gradient is its negative) and
 *                        grad_flow [2][H][W] (overwritten; taps outside the field get nothing, as zero
 *                        padding implies).  workspace: evk_warp_flow_grad_workspace_bytes() bytes,
 *                        16-byte aligned (2x2-block accumulators for the flow gradient).
 *   evk_voxel_grad_f32   gradient of evk_voxel_f32 / _aos_f32 (nearest, EVK_AUTO_SPAN), evk_voxel_negpos_f32 and
 *                        evk_voxel_windows_f32 (EVK_WINDOW_PAIRS), i.e. of events_to_voxel_torch voxel_grid.py:114-153,
 *                        events_to_neg_pos_voxel_torch :155-182 and the windows of voxel_grids_fixed_n/_t_torch
 *                        :37-80 and events_to_voxel_timesync_torch :82-112.  pairs: n_windows (start, end) int64
 *                        pairs on the device, or NULL for the one window [0, n).  Each window has its own
 *                        t0 = t[start], dt = t[end-1] - t0 and tn = ((t - t0) / dt) * (B-1) in f32, as the forward.
 *                        grad_out: [n_windows][B][H][W], or [n_windows][2][B][H][W] with EVK_WINDOW_NEGPOS (the
 *                        [p>0] / [p<=0] split; not EVK_NEGPOS_TRUTHY).  With g = grad_out at the event's pixel
 *                        (truncated, negative indices wrap), v_b = 1 - |tn - b| and torch's subgradients
 *                        (sign(0) = 0, a tie of max(0, v) splits the gradient in half):
 *                          grad_p = sum_b g[b] max(0, v_b)               (not written with EVK_WINDOW_NEGPOS)
 *                          G      = p sum_b g[b] s_b,  s_b = -sign(tn-b) (v_b > 0), -sign(tn-b)/2 (v_b == 0), 0 (v_b < 0)
 *                          grad_t = G (B-1) / dt, plus ((sum G tn) - (B-1) sum G) / dt at t[start] and
 *                                   -(sum G tn) / dt at t[end-1] of each window (sums in f64, on the device)
 *                        Finite events visit bins floor(tn)-1 .. floor(tn)+2 (the last only ties, when tn - b rounds
 *                        to -1 just below an integer); non-finite tn or p visit every bin, so NaN lands where
 *                        autograd puts it.
 *                        Events outside the grid, and with pairs those outside every window, get 0.  Windows that
 *                        share events need EVK_WINDOW_OVERLAP (the gradients are then added atomically).  With
 *                        EVK_EVENTS_AOS, x is the (N,4) record array of evk_voxel_aos_f32.
 *                        workspace: evk_voxel_grad_workspace_bytes() bytes, 256-byte aligned (the per-window sums
 *                        and grad_out re-laid out pixel-major).  Nothing is read back to the host.
 * --------------------------------------------------------------------------------------------- */
int evk_image_grad_f32(const float *x, const float *y, const float *p, int64_t n, int Himg, int Wimg,
                       float clipx, float clipy, unsigned flags, const float *grad_img, float *grad_x,
                       float *grad_y, float *grad_p, void *stream);
size_t evk_timestamp_image_grad_workspace_bytes(int Himg, int Wimg);
int evk_timestamp_image_grad_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                                 float t_first, float t_last, int Himg, int Wimg, float clipx, float clipy,
                                 unsigned flags, const float *grad_pos, const float *grad_neg,
                                 const float *out_pos, const float *out_neg, const float *cnt_pos,
                                 const float *cnt_neg, float *grad_x, float *grad_y, float *grad_t,
                                 double *sums, void *workspace, size_t workspace_bytes, void *stream);
size_t evk_warp_flow_grad_workspace_bytes(int H, int W);
int evk_warp_flow_grad_f32(const float *x, const float *y, const float *t, int64_t n, const float *flow,
                           int H, int W, float t0, const float *grad_xw, const float *grad_yw, float *grad_x,
                           float *grad_y, float *grad_t, float *grad_flow, double *sum_grad_t,
                           void *workspace, size_t workspace_bytes, void *stream);
size_t evk_voxel_grad_workspace_bytes(int n_windows, int B, int H, int W, unsigned flags);
int evk_voxel_grad_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                       const int64_t *pairs, int n_windows, int B, int H, int W, unsigned flags,
                       const float *grad_out, float *grad_p, float *grad_t, void *workspace,
                       size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Contrast maximisation, fused: linvel warp -> bounds mask -> bilinear IWE (+ derivative
 * images) -> Gaussian blur -> variance objective (+ analytic gradient).
 * Replaces variance_objective.evaluate_function / evaluate_gradient,
 * lib/contrast_max/objectives.py:211-264, i.e. get_iwe :165-199, linvel_warp.warp warps.py:51-61,
 * events_bounds_mask event_util.py:15-28, events_to_image_drv image.py:162-217,
 * scipy gaussian_filter + np.var / np.mean objectives.py:233-234,253-262.
 *   x,y,t,p : n doubles each (the reference API hands f64 numpy arrays) -- `_f64`, parity mode
 *             n floats each, t already relative to t_ref  -- `_f32`, fast mode
 *   (Hm,Wm) : img_size of the bounds mask;  (Hs,Ws): sensor size of the IWE canvas, which is
 *             (Hs+1)x(Ws+1); the reference always uses (180,240) (objectives.py:191-192).
 *   result  : 8 doubles on the device: f, g[0], g[1], sum(IWE), #events indexing outside the
 *             canvas (the reference's IndexError), var, and the un-mixed 2-D gradient (2)
 *             (g = 0 without EVK_CMAX_WANT_GRAD)
 *   iwe_out : optional (Hs+1)*(Ws+1) floats (the un-blurred IWE), diwe_out optional 2x that.
 *   p_scale : polarity multiplier (1, or 100 for the adaptive-lifespan branch objectives.py:225)
 *   workspace: evk_cmax_workspace_bytes(Hs,Ws) bytes of device scratch, 256-byte aligned.
 *   sigma   : the Gaussian blur of the image, scipy's gaussian_filter (truncate 4, mode 'reflect'), radius
 *             (int)(4 sigma + 0.5).  sigma <= 0: no blur.  NaN: EVK_E_ARG.  A radius above 64 (sigma >= 16.125,
 *             +inf included): EVK_E_UNSUPPORTED.  The same rule holds for every entry point below that takes a
 *             sigma, and each checks it first, before any CUDA call.
 * --------------------------------------------------------------------------------------------- */
size_t evk_cmax_workspace_bytes(int Hs, int Ws);
int evk_cmax_linvel_variance_f64(const double *x, const double *y, const double *t, const double *p,
                                 int64_t n, double p_scale, double vx, double vy, double t_ref,
                                 int Hm, int Wm, int Hs, int Ws, double sigma, unsigned flags,
                                 double *result,
                                 float *iwe_out, float *diwe_out, void *workspace,
                                 size_t workspace_bytes, void *stream);
int evk_cmax_linvel_variance_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                 int64_t n, float p_scale, float vx, float vy, int Hm, int Wm, int Hs,
                                 int Ws,
                                 double sigma, unsigned flags, double *result, float *iwe_out,
                                 float *diwe_out, void *workspace, size_t workspace_bytes,
                                 void *stream);

/* The reference's other objective functions on the same fused event pass (row f3).  `objective` is
 * one of EVK_OBJ_*; `obj_param` is the ISOA threshold / the SOSA exponent p.  result: 12 doubles --
 * [0] f, [1..2] g, [3] sum(IWE), [4] events outside the canvas, [5] mean(G), [6..7] un-mixed gradient,
 * [8] mean(G^2), [9] sum(exp(-p G)), [10] max(G), [11] #(G > thresh)   (G = blurred IWE; 0 for EVK_OBJ_VARIANCE).
 *   EVK_OBJ_VARIANCE  variance_objective  objectives.py:202-264   (result as documented above)
 *   EVK_OBJ_SOS       sos_ / rms_objective objectives.py:266-357   f = -mean(G^2), g = -mean(2 IWE * G3(dIWE))
 *   EVK_OBJ_SOE       soe_objective       objectives.py:358-400   f = -mean(exp G), g = -mean(exp(G) G3(dIWE))
 *   EVK_OBJ_MOA       moa_objective       objectives.py:401-430   f = -max(G), no gradient
 *   EVK_OBJ_ISOA      isoa_objective      objectives.py:431-477   f = +#(G > thresh), g = -sum([G>thresh] G3(dIWE))
 *   EVK_OBJ_SOSA      sosa_objective      objectives.py:478-523   f = -sum(exp(-p G)), g = -sum(-p exp(-p G) G3(dIWE)) */
#define EVK_OBJ_VARIANCE 0
#define EVK_OBJ_SOS 1
#define EVK_OBJ_SOE 2
#define EVK_OBJ_MOA 3
#define EVK_OBJ_ISOA 4
#define EVK_OBJ_SOSA 5
int evk_cmax_linvel_objective_f64(const double *x, const double *y, const double *t, const double *p,
                                  int64_t n, double p_scale, double vx, double vy, double t_ref,
                                  int Hm, int Wm, int Hs, int Ws, double sigma, unsigned flags,
                                  int objective, double obj_param, double *result, float *iwe_out,
                                  float *diwe_out, void *workspace, size_t workspace_bytes,
                                  void *stream);
int evk_cmax_linvel_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                  int64_t n, float p_scale, float vx, float vy, int Hm, int Wm,
                                  int Hs, int Ws, double sigma, unsigned flags, int objective,
                                  double obj_param, double *result, float *iwe_out, float *diwe_out,
                                  void *workspace, size_t workspace_bytes, void *stream);
/* K parameter candidates in ONE pass over the events (grid_search_initial, events_cmax.py:241-311,
 * evaluates num_samples^dims = 25 points per level): every event is read once and splatted into K
 * accumulators; results: 12 doubles per candidate (layout above).  params_host: K (vx,vy) pairs in
 * HOST memory, 1 <= K <= 32. */
int evk_cmax_linvel_objective_batch_f64(const double *x, const double *y, const double *t, const double *p,
                                        int64_t n, double p_scale, const double *params_host, int n_params,
                                        double t_ref, int Hm, int Wm, int Hs, int Ws, double sigma,
                                        unsigned flags, int objective, double obj_param, double *results,
                                        void *workspace, size_t workspace_bytes, void *stream);
int evk_iwe_objective_f32(const float *iwe, const float *diwe, int Hc, int Wc, double sigma,
                          unsigned flags, int objective, double obj_param, double *result,
                          void *workspace, size_t workspace_bytes, void *stream);

/* Rotation and 4-DoF motion models: the reference declares xyztheta_warp and pure_rotation_warp
 * (lib/contrast_max/warps.py:63-83) with empty warp(); contrast_max/warps.py defines them.  Same
 * event pass as the linvel entries for the IWE (get_iwe objectives.py:184-192, events_bounds_mask
 * event_util.py:26-27, events_to_image_drv image.py:179-217), then the objective of
 * objectives.py:202-523 and, with EVK_CMAX_WANT_GRAD, its exact gradient from a SECOND pass over
 * the events that gathers W = G(C) (C = the objective's coefficient image) at each event's four
 * taps -- no derivative images are formed (interpolate_to_derivative_img image.py:131-135 is only
 * contracted with W).  The gradient is not mixed across parameters (scipy's 3-D blur of the stack,
 * objectives.py:253, has no meaning for a stack of other than 2 channels).
 *   warp   : EVK_WARP_ROTATION,  model (host) = {cx, cy, omega}                 (dims 3)
 *            EVK_WARP_XYZTHETA,  model (host) = {hx, hy, hz, theta, cx, cy}     (dims 4)
 *   other arguments as evk_cmax_linvel_objective_*; the gradient pass needs (Hs+1)(Ws+1) <= 51200.
 *   result : 16 doubles -- [0] f, [1..4] g (zero past dims), [5] sum(IWE), [6] events outside the
 *            canvas, [7] mean(G), [8] mean(G^2), [9] sum(exp(-p G)), [10] max(G), [11] #(G > thresh).
 *   iwe_out: optional (Hs+1)*(Ws+1) floats (the un-blurred IWE). */
#define EVK_WARP_ROTATION 1
#define EVK_WARP_XYZTHETA 2
int evk_cmax_warp_objective_f64(const double *x, const double *y, const double *t, const double *p,
                                int64_t n, double p_scale, int warp, const double *model,
                                double t_ref, int Hm, int Wm, int Hs, int Ws, double sigma,
                                unsigned flags, int objective, double obj_param, double *result,
                                float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_warp_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                int64_t n, float p_scale, int warp, const double *model, int Hm,
                                int Wm, int Hs, int Ws, double sigma, unsigned flags, int objective,
                                double obj_param, double *result, float *iwe_out, void *workspace,
                                size_t workspace_bytes, void *stream);
/* Up to 32 models per pass over the events, f only (grid_search_initial, events_cmax.py:241-311,
 * samples 5^dims points per level): models_host = n_models consecutive models (3 or 6 doubles
 * each, HOST memory); results: 16 doubles per model (layout above, g = 0).  result[6] counts the
 * out-of-canvas events of all models together. */
int evk_cmax_warp_objective_batch_f64(const double *x, const double *y, const double *t,
                                      const double *p, int64_t n, double p_scale, int warp,
                                      const double *models_host, int n_models, double t_ref, int Hm,
                                      int Wm, int Hs, int Ws, double sigma, unsigned flags,
                                      int objective, double obj_param, double *results,
                                      void *workspace, size_t workspace_bytes, void *stream);

/* scipy.ndimage.gaussian_filter(img, sigma) for a 2-D f32 image (truncate=4, mode='reflect', f64 line
 * accumulation, f32 store after each axis) -- the blur every objective applies (objectives.py:233 ...).
 * tmp: H*W floats of scratch; out may not alias img.  sigma <= 0 copies img; NaN and radii above 64 are rejected
 * (the sigma rule above). */
int evk_gaussian_blur_f32(const float *img, int H, int W, double sigma, float *out, float *tmp, void *stream);

/* The objective (and gradient) of a PRECOMPUTED image of warped events, i.e. the iwe= / d_iwe=
 * form of evaluate_function / evaluate_gradient (objectives.py:211-264 with iwe given; used by
 * grid_cmax, events_cmax.py:68-70).  iwe: [Hc][Wc] f32, diwe: [2][Hc][Wc] f32 or NULL. */
int evk_variance_objective_f32(const float *iwe, const float *diwe, int Hc, int Wc, double sigma,
                               unsigned flags, double *result, void *workspace,
                               size_t workspace_bytes, void *stream);

/* Cross-GPU barrier on a stream, for the fused peer kernels.  peer_slots[r] = rank r's array of `world` 32-bit slots, mapped
 * on every rank (symmetric memory), zero before the first barrier; `epoch` = 1, 2, 3, ... (the caller counts).  Rank `rank`
 * stores `epoch` into slot [rank] of every rank and waits until all its own slots have reached it. */
int evk_peer_barrier(unsigned *const *peer_slots, int world, int rank, unsigned epoch, void *stream);

/* Sharded contrast maximisation, one process per GPU (SURVEY 8e): the all-reduce of the partial images is FUSED into the
 * objective kernel over NVLink peer memory -- no NCCL call, no host synchronisation between the two halves.
 *   evk_cmax_linvel_partial_*  event pass of THIS rank's shard; leaves its planar partial images images_out[3][Hs+1][Ws+1]
 *                              (IWE, dIWE/dvx, dIWE/dvy; objectives.py:184-192) and its out-of-canvas event count.
 *                              images_out / oob_out live in memory every rank has mapped (symmetric memory).
 *   (a cross-GPU barrier)
 *   evk_cmax_peer_tail_f32     every rank reads ALL ranks' partial images through peer pointers, sums them in rank order
 *                              while it gathers its tiles, blurs, reduces and writes f, g (objectives.py:231-264) --
 *                              bit-identical on all ranks.  result[4] = total out-of-canvas events. */
int evk_cmax_linvel_partial_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                double p_scale, double vx, double vy, double t_ref, int Hm, int Wm, int Hs, int Ws,
                                unsigned flags, float *images_out, unsigned long long *oob_out, void *workspace,
                                size_t workspace_bytes, void *stream);
int evk_cmax_linvel_partial_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n,
                                float p_scale, float vx, float vy, int Hm, int Wm, int Hs, int Ws, unsigned flags,
                                float *images_out, unsigned long long *oob_out, void *workspace,
                                size_t workspace_bytes, void *stream);
int evk_cmax_peer_tail_f32(const float *const *peer_images, const unsigned long long *const *peer_oob, int world,
                           int Hc, int Wc, double sigma, unsigned flags, double *result, void *workspace,
                           size_t workspace_bytes, void *stream);

/* Objective only (f) for a dense-flow warp: warp_events_flow_torch + bilinear IWE
 * (lib/visualization/draw_flow.py:18-21) + the variance objective.  flow: [2][Hs][Ws]. */
int evk_cmax_flow_variance_f32(const float *x, const float *y, const float *t, const float *p,
                               int64_t n, const float *flow, float t0, int Hs, int Ws, double sigma,
                               unsigned flags, double *result, float *iwe_out, void *workspace,
                               size_t workspace_bytes, void *stream);

/* Dense-flow contrast maximisation over a batch of samples, as a differentiable loss: the reference's
 * motion_compensate (lib/visualization/draw_flow.py:15-26: warp_events_flow_torch, then the bilinear
 * events_to_image_torch) followed by an objective of lib/contrast_max/objectives.py.  Sample b is the events
 * [offsets[b], offsets[b+1]) (clipped to [0, n_events); end < start is empty), warped by flow[b]:
 *   x' = x + u(x,y) t_rel,  y' = y + v(x,y) t_rel     (optic_flow.py:37-44; t_rel = t - t0[b], given)
 * The IWE of sample b is the bilinear splat of p on the (H+1)x(W+1) canvas of every event with 0 <= x' < W and
 * 0 <= y' < H (f32 comparisons); other events contribute nothing.  An event whose x' or y' is not finite makes the
 * whole IWE of its sample NaN, and so its f.  Then G = gaussian_filter(IWE, sigma) (sigma 0: no blur) and, P = (H+1)(W+1):
 *   EVK_OBJ_VARIANCE  f = -var(G)          EVK_OBJ_SOS   f = -mean(G^2)
 *   EVK_OBJ_SOE       f = -mean(exp G)     EVK_OBJ_SOSA  f = -sum(exp(-obj_param G))
 * (EVK_OBJ_MOA / EVK_OBJ_ISOA are piecewise constant: EVK_E_UNSUPPORTED.)
 *   x, y, t_rel, p : n_events floats;  offsets: batch+1 int64 on the device;  flow: [batch][2][H][W] f32
 *   f_out          : batch doubles;  iwe_out: [batch][H+1][W+1] floats, which the backward takes as `iwe`
 * evk_cmax_flow_objective_grad_f32 writes grad_flow [batch][2][H][W] = sum_b grad_f[b] df_b/dflow[b], the exact
 * derivative of the f above (grad_f: batch floats on the device): with W_b = G(grad_f[b] df_b/dG), per kept event
 *   df/dx' = p[(1-dy)(W01-W00) + dy(W11-W10)],  df/dy' = p[(1-dx)(W10-W00) + dx(W11-W01)]
 * times t_rel, spread over the four grid_sample taps of the event's (x, y); taps outside the field get nothing.
 * workspace: evk_cmax_flow_objective_workspace_bytes(batch, H, W) bytes, 256-byte aligned, for either call; 0 for
 * arguments the entries reject (the canvas of every batched entry is at most 2^30 pixels (H+1)(W+1)).
 * Neither call synchronises, and both launch the same kernels whatever the batch. */
size_t evk_cmax_flow_objective_workspace_bytes(int batch, int H, int W);
int evk_cmax_flow_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                const int64_t *offsets, int batch, int64_t n_events, const float *flow,
                                int H, int W, double sigma, int objective, double obj_param, double *f_out,
                                float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_flow_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                     const int64_t *offsets, int batch, int64_t n_events, const float *flow,
                                     int H, int W, double sigma, int objective, double obj_param,
                                     const float *iwe, const float *grad_f, float *grad_flow,
                                     void *workspace, size_t workspace_bytes, void *stream);

/* The dense-flow contrast objective with the flow of every sample given on a coarse grid of nodes (tile-based flow,
 * Shiba et al., ECCV 2022).  grid_flow: [batch][2][gh][gw] f32 on the device, 2 <= gh <= H, 2 <= gw <= W,
 * gh * gw <= 4096.  Node (i, j) sits at pixel (j (W-1)/(gw-1), i (H-1)/(gh-1)) (align_corners), and an event at
 * (x, y) takes the flow (u, v) = bilinear interpolation of grid_flow[b] at (x rx, y ry), rx = (gw-1)/(W-1) and
 * ry = (gh-1)/(H-1) rounded to f32, products in f32; a node tap outside the grid contributes 0 (zero padding, as the
 * grid_sample of optic_flow.py:37-44).  Everything after that is evk_cmax_flow_objective_f32: x' = x + u t_rel,
 * y' = y + v t_rel in f32, kept iff 0 <= x' < W and 0 <= y' < H, the bilinear IWE on the (H+1)x(W+1) canvas
 * (draw_flow.py:15-26), the blur, the four objectives (EVK_OBJ_MOA / EVK_OBJ_ISOA: EVK_E_UNSUPPORTED) and a NaN f for
 * a sample with a non-finite x' or y'.  For events at integer pixels inside the sensor, f equals the dense-flow f of
 * the flow that bilinear upsampling with align_corners makes of the nodes, to f32 rounding; at gh = H, gw = W the grid
 * is the dense flow.
 *   f_out: batch doubles;  iwe_out: [batch][H+1][W+1] floats, which the backward takes as `iwe`
 * evk_cmax_grid_flow_objective_grad_f32 writes grad_grid [batch][2][gh][gw] floats = grad_f[b] df_b/dgrid_flow[b]:
 * df/dx' and df/dy' of evk_cmax_flow_objective_grad_f32, times t_rel, spread over the event's four node taps with
 * their bilinear weights, summed per CTA in shared memory and across CTAs in f64, then rounded to f32.
 * workspace: evk_cmax_grid_flow_objective_workspace_bytes(batch, gh, gw, H, W) bytes, 256-byte aligned, for either
 * call; 0 for arguments the entries reject.  batch <= 65535.  Neither call synchronises, and both launch the same
 * kernels whatever the batch. */
size_t evk_cmax_grid_flow_objective_workspace_bytes(int batch, int gh, int gw, int H, int W);
int evk_cmax_grid_flow_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                     const int64_t *offsets, int batch, int64_t n_events, const float *grid_flow,
                                     int gh, int gw, int H, int W, double blur_sigma, int objective, double obj_param,
                                     double *f_out, float *iwe_out, void *workspace, size_t workspace_bytes,
                                     void *stream);
int evk_cmax_grid_flow_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                          const int64_t *offsets, int batch, int64_t n_events,
                                          const float *grid_flow, int gh, int gw, int H, int W, double blur_sigma,
                                          int objective, double obj_param, const float *iwe, const float *grad_f,
                                          float *grad_grid, void *workspace, size_t workspace_bytes, void *stream);

/* Many node grids per sample in one pass over the events (a batched line search of a grid-flow fit):
 * f_out[b][j] is exactly the f_b of evk_cmax_grid_flow_objective_f32 with grid_flow[b] = cand[b][j].
 *   cand : [batch][n_cand][2][gh][gw] floats on the device, 1 <= n_cand <= 32, n_cand * gh * gw <= 12288 (the
 *          candidate grids of a sample fit in shared memory), batch * n_cand <= 65535
 *   f_out: [batch][n_cand] doubles
 * Every event is read once; its node cell and weights are computed once and used for every candidate.  All limits are
 * checked before any CUDA call.  Forward only.  workspace: evk_cmax_grid_flow_candidates_workspace_bytes(batch,
 * n_cand, gh, gw, H, W) bytes, 256-byte aligned; 0 for arguments the entry rejects.  The call does not synchronise
 * and launches the same kernels whatever batch and n_cand. */
size_t evk_cmax_grid_flow_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W);
int evk_cmax_grid_flow_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                      const int64_t *offsets, int batch, int64_t n_events, const float *cand,
                                      int n_cand, int gh, int gw, int H, int W, double blur_sigma, int objective,
                                      double obj_param, double *f_out, void *workspace, size_t workspace_bytes,
                                      void *stream);

/* Depth from a known camera motion: the contrast objective of evk_cmax_motion_depth_objective_f32 with
 * EVK_WARP_CAMERA_MOTION, where the inverse depth of every event is interpolated from a gh x gw grid of nodes of its
 * sample instead of read from an array.
 *   motion        : [batch][8] doubles on the device, the rows (wx, wy, wz, vx, vy, vz, fx, fy) of the camera motion
 *                   (data: they get no gradient), principal point (cx, cy)
 *   inv_depth_grid: [batch][gh][gw] f32 on the device, 2 <= gh <= H, 2 <= gw <= W, gh * gw <= 4096
 * Node (i, j) sits at pixel (j (W-1)/(gw-1), i (H-1)/(gh-1)) (align_corners), and an event at (x, y) takes
 * rho = bilinear interpolation of inv_depth_grid[b] at (x rx, y ry), with the node cell, weights, f32 products and
 * zero outside taps of evk_cmax_grid_flow_objective_f32.  Everything after that is the camera motion's: the keep rules
 * (a negative or non-finite rho, Pz <= 0 or a non-finite Pz: not kept), the warp, the bounds mask, the splat on the
 * (H+1)x(W+1) canvas, the blur and the four objectives (EVK_OBJ_MOA / EVK_OBJ_ISOA: EVK_E_UNSUPPORTED).  The rotation
 * exp([theta]x) b of an event is computed once per pass, then the translation and projection per candidate, in
 * the camera motion's order of operations, so every event's taps are the camera motion's bit for bit: at gh = H,
 * gw = W with events at integer pixels rho is the node and f is evk_cmax_motion_depth_objective_f32's with that rho, and
 * at v = 0 f is EVK_WARP_CAMERA_ROTATION's, up to the order in which the f32 image sums add the taps.
 *   f_out: batch doubles;  iwe_out: [batch][H+1][W+1] floats, which the backward takes as `iwe`
 * evk_cmax_depth_grid_objective_grad_f32 writes grad_grid [batch][gh][gw] floats = grad_f[b] df_b/dinv_depth_grid[b]:
 * per kept event df/dx' and df/dy' of evk_cmax_motion_objective_grad_f32 times
 *   dx'/drho = d fx iz (vx - X vz),  dy'/drho = d fy iz (vy - Y vz)   (d = t_rel)
 * spread over the event's four node taps with their bilinear weights, summed per CTA in shared memory and across CTAs
 * in f64, then rounded to f32.  At v = 0 the gradient is exactly zero.
 * workspace: evk_cmax_depth_grid_objective_workspace_bytes(batch, gh, gw, H, W) bytes (what the grid flow's query
 * returns), 256-byte aligned, for either call; 0 for arguments the entries reject.  batch <= 65535.  Neither call
 * synchronises, and both launch the same kernels whatever the batch. */
size_t evk_cmax_depth_grid_objective_workspace_bytes(int batch, int gh, int gw, int H, int W);
int evk_cmax_depth_grid_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                      const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                      double cx, double cy, const float *inv_depth_grid, int gh, int gw, int H, int W,
                                      double blur_sigma, int objective, double obj_param, double *f_out,
                                      float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_depth_grid_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                           const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                           double cx, double cy, const float *inv_depth_grid, int gh, int gw, int H,
                                           int W, double blur_sigma, int objective, double obj_param,
                                           const float *iwe, const float *grad_f, float *grad_grid, void *workspace,
                                           size_t workspace_bytes, void *stream);

/* Many inverse-depth grids per sample in one pass over the events: f_out[b][j] is exactly the f_b of
 * evk_cmax_depth_grid_objective_f32 with inv_depth_grid[b] = cand[b][j].
 *   cand : [batch][n_cand][gh][gw] floats on the device, 1 <= n_cand <= 32, n_cand * gh * gw <= 12288 (the limit of
 *          the grid flow, 48 KB of f32 nodes here), batch * n_cand <= 65535
 *   f_out: [batch][n_cand] doubles
 * Every event is read once; its node cell, weights and rotation are computed once and used for every candidate.  All
 * limits are checked before any CUDA call.  Forward only.  workspace: evk_cmax_depth_grid_candidates_workspace_bytes(
 * batch, n_cand, gh, gw, H, W) bytes, 256-byte aligned; 0 for arguments the entry rejects.  The call does not
 * synchronise and launches the same kernels whatever batch and n_cand. */
size_t evk_cmax_depth_grid_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W);
int evk_cmax_depth_grid_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                       double cx, double cy, const float *cand, int n_cand, int gh, int gw, int H,
                                       int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                       void *workspace, size_t workspace_bytes, void *stream);

/* Camera motion and depth together: the joint backward of evk_cmax_depth_grid_objective_f32, whose f it leaves as it is.
 * The arguments are those of evk_cmax_depth_grid_objective_grad_f32, and it writes, besides the same grad_grid,
 *   grad_motion: [batch][6] doubles = grad_f[b] df_b/d(wx, wy, wz, vx, vy, vz) (the focal lengths and the principal
 *                point are constants)
 * per kept event df/dx' and df/dy' of evk_cmax_motion_objective_grad_f32 contracted with the f32 Jacobian rows of
 * EVK_WARP_CAMERA_MOTION at the event's interpolated rho, in f64, summed per CTA and across CTAs in f64: the first six
 * components of evk_cmax_motion_depth_objective_grad_f32's gradient at that rho, up to the order of the sums.
 * workspace: evk_cmax_depth_grid_joint_grad_workspace_bytes(batch, gh, gw, H, W) bytes (the depth grid's), 256-byte
 * aligned; 0 for arguments the entry rejects.  The call does not synchronise. */
size_t evk_cmax_depth_grid_joint_grad_workspace_bytes(int batch, int gh, int gw, int H, int W);
int evk_cmax_depth_grid_joint_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                       double cx, double cy, const float *inv_depth_grid, int gh, int gw, int H, int W,
                                       double blur_sigma, int objective, double obj_param, const float *iwe,
                                       const float *grad_f, float *grad_grid, double *grad_motion, void *workspace,
                                       size_t workspace_bytes, void *stream);

/* Many (motion, inverse-depth grid) pairs per sample in one pass over the events: f_out[b][j] is exactly the f_b of
 * evk_cmax_depth_grid_objective_f32 with motion row [b] = motion[b][j] and inv_depth_grid[b] = cand[b][j].
 *   motion: [batch][n_cand][8] doubles on the device, rows (wx, wy, wz, vx, vy, vz, fx, fy)
 *   cand  : [batch][n_cand][gh][gw] floats; the limits of evk_cmax_depth_grid_candidates_f32 (1 <= n_cand <= 32,
 *           n_cand * gh * gw <= 12288, batch * n_cand <= 65535), checked before any CUDA call
 *   f_out : [batch][n_cand] doubles
 * Every event is read once and its node cell computed once; the rotation is computed per candidate.  Forward only.
 * workspace: evk_cmax_depth_grid_joint_candidates_workspace_bytes(batch, n_cand, gh, gw, H, W) bytes (the depth grid
 * candidates'), 256-byte aligned; 0 for arguments the entry rejects.  The call does not synchronise. */
size_t evk_cmax_depth_grid_joint_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W);
int evk_cmax_depth_grid_joint_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                             const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                             double cx, double cy, const float *cand, int n_cand, int gh, int gw, int H,
                                             int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                             void *workspace, size_t workspace_bytes, void *stream);

/* Parametric contrast maximisation over a batch of samples, as a differentiable loss: per sample the f32
 * fast-mode evaluation of evk_cmax_warp_objective_f32 / evk_cmax_linvel_objective_f32 with Hm = Hs = H,
 * Wm = Ws = W, p_scale 1 and no flags (get_iwe, lib/contrast_max/objectives.py:184-192).  Sample b is the
 * events [offsets[b], offsets[b+1]) (clipped to [0, n_events); end < start is empty), warped by its own
 * parameters params[b] (K doubles, in DEVICE memory) with the model `warp`:
 *   EVK_WARP_LINVEL    (vx, vy)                K = 2   x' = x - t_rel vx (lib/contrast_max/warps.py:51-61)
 *   EVK_WARP_ROTATION  (cx, cy, omega)         K = 3
 *   EVK_WARP_XYZTHETA  (hx, hy, hz, theta)     K = 4   about the centre (cx, cy) given here
 *   EVK_WARP_AFFINE    (hx, hy, a11, a12, a21, a22)            K = 6   about (cx, cy)
 *   EVK_WARP_HOMOGRAPHY (hx, hy, a11, a12, a21, a22, g1, g2)   K = 8   about (cx, cy)
 *   EVK_WARP_CAMERA_ROTATION (wx, wy, wz, fx, fy)              K = 5   principal point (cx, cy)
 * (cx, cy) is the fixed centre of xyztheta, affine and homography and the principal point of the camera rotation,
 * and is ignored by the other models.  With
 * d = t_rel, u = x - cx, v = y - cy, the two planar models are first order in d:
 *   affine:      sx = (hx + a11 u) + a12 v,  sy = (hy + a22 v) + a21 u,  x' = x - d sx,  y' = y - d sy
 *   homography:  sx, sy as affine, nx = u - d sx, ny = v - d sy, q = d ((g1 u) + (g2 v)), w = 1 - q,
 *                x' = (x - d sx) + nx q / w,  y' = (y - d sy) + ny q / w
 * An event whose w is <= 0 or not finite (past the homography's horizon) is not kept.  Affine at
 * (hx, hy, hz, -theta, theta, hz) is xyztheta bit for bit, and homography at g1 = g2 = 0 is affine bit for bit.
 * The camera rotation is exact in the rotation: w = (wx, wy, wz) is the camera's angular velocity (rad/s) in its own
 * frame (x right, y down, z along the optical axis), fx, fy its focal lengths (px, no skew), and x, y undistorted:
 *   b = ((x - cx) / fx, (y - cy) / fy, 1),  theta = d w,  phi = |theta|,  c = theta x b,  e = theta x c,
 *   P = exp([theta]x) b = (b + A c) + B e,  A = sin(phi) / phi,  B = (1 - cos(phi)) / phi^2,
 *   x' = cx + fx (Px iz),  y' = cy + fy (Py iz),  iz = 1 / Pz
 * with A = r cos(phi/2), B = r^2 / 2, r = sin(phi/2) / (phi/2) (1 at phi = 0).  An event with Pz <= 0 or a non-finite
 * Pz has rotated behind the camera and is not kept.  With fx = fy, w = (0, 0, wz) is EVK_WARP_ROTATION (cx, cy, -wz).
 * grad_params carries the exact derivatives of all five values, the focal lengths included.
 * All in f32, in the order written.  An event is kept iff 0 < x' <= W and 0 < y' <= H (events_bounds_mask,
 * lib/util/event_util.py:26-27; NaN compares false and is kept, then contributes nothing) and splatted
 * bilinearly on the (H+1)x(W+1) canvas (events_to_image_drv, lib/representations/image.py:179-217).  Then
 * G = gaussian_filter(IWE, sigma) and f is one of the four objectives of evk_cmax_flow_objective_f32
 * (EVK_OBJ_MOA / EVK_OBJ_ISOA: EVK_E_UNSUPPORTED).
 *   f_out   : batch doubles;  iwe_out: [batch][H+1][W+1] floats, which the backward takes as `iwe`
 * evk_cmax_motion_objective_grad_f32 writes grad_params [batch][K] doubles = grad_f[b] df_b/dparams[b], the
 * exact derivative of the f above with the floor and keep decisions held (grad_f: batch floats on the device):
 * with W_b = G(grad_f[b] df_b/dG), per kept event
 *   df/dparams_k += p[(1-dy)(W01-W00) + dy(W11-W10)] dx'/dparams_k + p[(1-dx)(W10-W00) + dx(W11-W01)] dy'/dparams_k
 * For linvel this is not the reference's evaluate_gradient (objectives.py:251-264), which mixes the two
 * channels in its 3-D blur and multiplies by the un-blurred IWE.  No limit on the canvas size.
 * workspace: evk_cmax_motion_objective_workspace_bytes(batch, H, W) bytes, 256-byte aligned, for either call; 0 for
 * arguments the entries reject (the canvas of every batched entry is at most 2^30 pixels (H+1)(W+1)).
 * Neither call synchronises, and both launch the same kernels whatever the batch. */
#define EVK_WARP_LINVEL 3
#define EVK_WARP_AFFINE 4
#define EVK_WARP_HOMOGRAPHY 5
#define EVK_WARP_CAMERA_ROTATION 6
size_t evk_cmax_motion_objective_workspace_bytes(int batch, int H, int W);
int evk_cmax_motion_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                  const int64_t *offsets, int batch, int64_t n_events, int warp,
                                  const double *params, int K, double cx, double cy, int H, int W,
                                  double sigma, int objective, double obj_param, double *f_out,
                                  float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_motion_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, int warp,
                                       const double *params, int K, double cx, double cy, int H, int W,
                                       double sigma, int objective, double obj_param, const float *iwe,
                                       const float *grad_f, double *grad_params, void *workspace,
                                       size_t workspace_bytes, void *stream);

/* Many parameter vectors per sample in one pass over the events: the sample points of a grid search per window
 * (grid_search_initial, lib/contrast_max/events_cmax.py:241-311) or the step lengths of a batched line search.
 * f_out[b][j] is exactly the f_b of evk_cmax_motion_objective_f32 with params[b] = cand[b][j] (get_iwe,
 * lib/contrast_max/objectives.py:184-192): the same warp, keep rule, splat, blur and objectives, the same argument
 * checks (EVK_OBJ_MOA / EVK_OBJ_ISOA: EVK_E_UNSUPPORTED) and the blur-sigma rule for blur_sigma (0 or less: no blur;
 * NaN: EVK_E_ARG; a radius over 64: EVK_E_UNSUPPORTED), all checked before any CUDA call.  Forward only: no image out,
 * no gradient.
 *   cand : [batch][n_cand][K] doubles in DEVICE memory, 1 <= n_cand <= 32, batch * n_cand <= 65535
 *   f_out: [batch][n_cand] doubles
 * Every event is read once and splatted under each of its sample's n_cand candidates.
 * workspace: evk_cmax_motion_candidates_workspace_bytes(batch, n_cand, H, W) bytes (about 28 bytes per canvas pixel
 * and candidate), 256-byte aligned; the query returns 0 for arguments the entry rejects.
 * The call does not synchronise and launches the same kernels whatever batch and n_cand. */
size_t evk_cmax_motion_candidates_workspace_bytes(int batch, int n_cand, int H, int W);
int evk_cmax_motion_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                   const int64_t *offsets, int batch, int64_t n_events, int warp,
                                   const double *cand, int n_cand, int K, double cx, double cy, int H, int W,
                                   double blur_sigma, int objective, double obj_param, double *f_out,
                                   void *workspace, size_t workspace_bytes, void *stream);

/* Camera motion with known depth: the three entries above for the model EVK_WARP_CAMERA_MOTION, whose warp needs the
 * inverse depth of every event.  Each has the signature of its depth-free twin with inv_depth inserted right after p:
 *   inv_depth: n_events floats on the device, rho = 1 / Z of the event's scene point at the event's time (Z along the
 *              optical axis, in the depth unit of v)
 * and accepts warp = EVK_WARP_CAMERA_MOTION only (any other code: EVK_E_ARG), with K = 8 and rows
 *   EVK_WARP_CAMERA_MOTION (wx, wy, wz, vx, vy, vz, fx, fy)    K = 8   principal point (cx, cy)
 * w is the camera's angular velocity (rad/s) in its own frame (x right, y down, z along the optical axis), v its linear
 * velocity in the camera frame at t0 (depth units per second), fx, fy its focal lengths (px, no skew), and x, y are
 * undistorted.  With d = t_rel and b, theta, phi, A, B exactly as in the camera rotation above:
 *   P = exp([theta]x) b + (rho d) v,  iz = 1 / Pz,  X = Px iz,  Y = Py iz,  x' = cx + fx X,  y' = cy + fy Y
 * exact for a camera whose pose at time t, in the camera frame at t0, is (exp(d [w]x), d v): it rotates at a constant
 * rate and moves at a constant velocity.  Keep rules: an event with Pz <= 0 or a non-finite Pz (behind the camera), or
 * with a negative or non-finite rho, is not kept (no contribution, no gradient); rho = 0 is a point at infinity.
 * Derivatives, with Q = exp([theta]x) b iz and the left Jacobian J_l = A I + B [theta]x + C theta theta^T of the camera
 * rotation:
 *   dx'/dw = -d fx J_l^T (X Qy, -(Qz + X Qx), Qy),     dy'/dw = -d fy J_l^T (Qz + Y Qy, -Y Qx, -Qx)
 *   dx'/dv = (rho d) fx iz (1, 0, -X),                 dy'/dv = (rho d) fy iz (0, 1, -Y)
 * and dx'/dfx, dy'/dfx, dx'/dfy, dy'/dfy those of the camera rotation with this P's iz, X and Y.  grad_params carries
 * all eight derivatives, the focal lengths included.  Identities: at v = 0 or rho = 0 the translation is an added exact
 * zero, so x', y', the images and f equal EVK_WARP_CAMERA_ROTATION's at (wx, wy, wz, fx, fy) bit for bit (the w
 * columns of the gradient to f32 rounding); at w = 0 the warp is the exact projective translation.  All in f32, in the
 * order written.  Everything else -- keep rule on the canvas, splat, blur, objectives, argument checks, images,
 * workspaces (the _workspace_bytes queries return what the twins' return), no synchronisation and a launch count
 * independent of the batch -- is the twin's. */
#define EVK_WARP_CAMERA_MOTION 7
size_t evk_cmax_motion_depth_objective_workspace_bytes(int batch, int H, int W);
int evk_cmax_motion_depth_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                        const float *inv_depth, const int64_t *offsets, int batch, int64_t n_events,
                                        int warp, const double *params, int K, double cx, double cy, int H, int W,
                                        double blur_sigma, int objective, double obj_param, double *f_out,
                                        float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_motion_depth_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                             const float *inv_depth, const int64_t *offsets, int batch,
                                             int64_t n_events, int warp, const double *params, int K, double cx,
                                             double cy, int H, int W, double blur_sigma, int objective, double obj_param,
                                             const float *iwe, const float *grad_f, double *grad_params,
                                             void *workspace, size_t workspace_bytes, void *stream);
size_t evk_cmax_motion_depth_candidates_workspace_bytes(int batch, int n_cand, int H, int W);
int evk_cmax_motion_depth_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                         const float *inv_depth, const int64_t *offsets, int batch, int64_t n_events,
                                         int warp, const double *cand, int n_cand, int K, double cx, double cy, int H,
                                         int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                         void *workspace, size_t workspace_bytes, void *stream);

/* Motion segmentation by motion compensation (Stoffregen, Gallego, Drummond, Kleeman, Scaramuzza, ICCV 2019):
 * n_models = M motion models per sample (1 <= M <= 8) and a soft membership weights[e][m] (n_events x M floats,
 * row-major, in DEVICE memory) of every event in every model.  Samples, t_rel, warp models, keep rule, canvas,
 * blur, objectives and argument checks are those of evk_cmax_motion_objective_f32.  Image (b, m) is the IWE of
 * sample b's events warped by params[b][m] (params: [batch][M][K] doubles on the device), every event splatted with
 * the f32 product p[e] * weights[e][m]: exactly the taps of evk_cmax_motion_objective_f32 run on p * weights[:, m]
 * and params[:, m].  f[b][m] is that image's objective; at M = 1 with weights 1 the entries compute what the motion
 * objective computes.  batch * M <= 65535 canvases.
 *   f_out  : [batch][M] doubles;  iwe_out: [batch][M][H+1][W+1] floats, which the backward and the assignment take
 * evk_cmax_motion_segment_grad_f32 (grad_f [batch][M] floats on the device) writes grad_params [batch][M][K] doubles,
 * the derivative of evk_cmax_motion_objective_grad_f32 per (b, m) with the event weights p * weights[e][m], and, when
 * grad_weights is not NULL, grad_weights [n_events][M] floats = sum_{b,m} grad_f[b][m] df[b][m] / dweights[e][m]:
 *   p[e] sum_taps k_tap dF/dI(tap)   (k the bilinear fractions of the event under params[b][m]; 0 when it is not
 *   kept).  The footprint comes from the unweighted taps, so an event of weight 0 (or p = 0) still has a weight
 *   gradient.  Only the rows of events inside a sample are written (the caller zeroes the others), so that a batch
 *   may run as several calls on chunks of its samples; samples must not overlap.
 * evk_cmax_motion_segment_candidates_f32 scores n_cand parameter vectors per model in one pass over the events:
 * f_out[b][m][j] is the f[b][m] of evk_cmax_motion_segment_f32 with params[b][m] = cand[b][m][j]
 * (cand: [batch][M][n_cand][K] doubles on the device; M * n_cand <= 32, batch * M * n_cand <= 65535).
 * evk_cmax_motion_segment_assign_f32 is the E-step: with G_bm the blurred iwe[b][m] (blur_sigma),
 *   c[e][m] = max(0, sum_taps k_tap G_bm(tap))  (k the polarity- and weight-free bilinear fractions under
 *   params[b][m]; 0 when the event is not kept under model m), then
 *   weights_out[e][m] = (c[e][m] + eps) / (sum_i c[e][i] + M eps)   (eps >= 0)
 * A row whose c are all 0 with eps = 0 is 1/M; a non-finite c makes its own row non-finite.  As for grad_weights,
 * only the rows of events inside a sample are written (motion_segmentation_assign_torch sets the others to 1/M).
 * workspace: evk_cmax_motion_segment_workspace_bytes(batch, M, H, W) bytes for the forward, the backward and the
 * assignment; evk_cmax_motion_segment_candidates_workspace_bytes(batch, M, n_cand, H, W) for the candidates.  Both
 * 256-byte aligned; the queries return 0 for arguments the entries reject.  Every argument is checked before any
 * CUDA call; no call synchronises, and each launches the same kernels whatever the batch. */
size_t evk_cmax_motion_segment_workspace_bytes(int batch, int n_models, int H, int W);
int evk_cmax_motion_segment_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                const float *weights, int n_models, const int64_t *offsets, int batch,
                                int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                int H, int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                float *iwe_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_cmax_motion_segment_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                     const float *weights, int n_models, const int64_t *offsets, int batch,
                                     int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                     int H, int W, double blur_sigma, int objective, double obj_param, const float *iwe,
                                     const float *grad_f, double *grad_params, float *grad_weights,
                                     void *workspace, size_t workspace_bytes, void *stream);
size_t evk_cmax_motion_segment_candidates_workspace_bytes(int batch, int n_models, int n_cand, int H, int W);
int evk_cmax_motion_segment_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                           const float *weights, int n_models, const int64_t *offsets, int batch,
                                           int64_t n_events, int warp, const double *cand, int n_cand, int K,
                                           double cx, double cy, int H, int W, double blur_sigma, int objective,
                                           double obj_param, double *f_out, void *workspace,
                                           size_t workspace_bytes, void *stream);
int evk_cmax_motion_segment_assign_f32(const float *x, const float *y, const float *t_rel, int n_models,
                                       const int64_t *offsets, int batch, int64_t n_events, int warp,
                                       const double *params, int K, double cx, double cy, int H, int W,
                                       const float *iwe, double blur_sigma, double eps, float *weights_out,
                                       void *workspace, size_t workspace_bytes, void *stream);

/* Dense-flow average-timestamp loss (Zhu et al., CVPR'19) over a batch of samples, as a differentiable loss:
 * warp_events_flow_torch (lib/transforms/optic_flow.py:5-46), then the timestamp images of
 * events_to_timestamp_image_torch (lib/representations/image.py:286-353) on the canvas of motion_compensate
 * (lib/visualization/draw_flow.py:15-26), blurred and squared as zhu_timestamp_objective does
 * (lib/contrast_max/objectives.py:524-551), with the sign of a loss to minimise.  Sample b is the events
 * [offsets[b], offsets[b+1]) (clipped to [0, n_events); end < start is empty), warped by flow[b] and kept exactly
 * as in evk_cmax_flow_objective_f32 (0 <= x' < W, 0 <= y' < H; a non-finite x' or y' makes the sample's f NaN).
 * tau is each event's normalised stamp, prepared by the caller: (t - t_first) / (t_last - t_first + 1e-6) of its
 * sample, or (-t + t_last) / (...) for the reversed images.  Per polarity s (p > 0 / p <= 0; a NaN p is dropped),
 * with k the bilinear tap weights of the kept events on the (H+1)x(W+1) canvas:
 *   T_s = S_s / C_s,  S_s = sum tau k,  C_s = 1 + sum k,   f_b = sum gaussian_filter(T_+, sigma)^2 + sum (...T_-...)^2
 * (sigma 0: no blur).
 *   x, y, t_rel, tau, p : n_events floats;  offsets: batch+1 int64 on the device;  flow: [batch][2][H][W] f32
 *   f_out: batch doubles;  ts_out, cnt_out: [batch][2][H+1][W+1] floats (T and C, polarity 0 positive), which the
 *   backward takes as ts_img, cnt_img.  0 <= batch <= 32767.
 * evk_flow_timestamp_objective_grad_f32 writes grad_flow [batch][2][H][W] = grad_f[b] df_b/dflow[b], the exact
 * derivative of the f above with the floor and keep decisions held (grad_f: batch floats on the device): with
 * U_s = G(2 grad_f[b] G_s), A_s = U_s / C_s and B_s = -U_s T_s / C_s, per kept event of polarity s and each of its
 * four taps q = tau A_s + B_s, and
 *   df/dx' = (1-dy)(q01-q00) + dy(q11-q10),  df/dy' = (1-dx)(q10-q00) + dx(q11-q01)
 * times t_rel, spread over the four grid_sample taps of the event's (x, y); taps outside the field get nothing.
 * workspace: evk_flow_timestamp_objective_workspace_bytes(batch, H, W) bytes, 256-byte aligned, for either call; 0 for
 * arguments the entries reject (the canvas of every batched entry is at most 2^30 pixels (H+1)(W+1)).
 * Neither call synchronises, and both launch the same kernels whatever the batch. */
size_t evk_flow_timestamp_objective_workspace_bytes(int batch, int H, int W);
int evk_flow_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                     const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                     const float *flow, int H, int W, double sigma, double *f_out, float *ts_out,
                                     float *cnt_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_flow_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                          const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                          const float *flow, int H, int W, double sigma, const float *ts_img,
                                          const float *cnt_img, const float *grad_f, float *grad_flow,
                                          void *workspace, size_t workspace_bytes, void *stream);

/* Parametric average-timestamp loss (Zhu et al., CVPR'19) over a batch of samples, as a differentiable loss: the
 * reference's zhu_timestamp_objective (lib/contrast_max/objectives.py:524-558), driven by its warp_function, with the
 * sign of a loss to minimise.  Sample b is the events [offsets[b], offsets[b+1]) (clipped to [0, n_events); end < start
 * is empty), warped by its own parameters params[b] (K doubles in DEVICE memory) with the model `warp` and its f32
 * arithmetic exactly as in evk_cmax_motion_objective_f32 (EVK_WARP_LINVEL / _ROTATION / _XYZTHETA / _AFFINE /
 * _HOMOGRAPHY / _CAMERA_ROTATION; the centre (cx, cy) of xyztheta and the planar models, the principal point of the
 * camera rotation, whose events behind the camera are not kept).  An event contributes iff its splat in that loss is not zero: x', y' finite, 0 < x' < W and
 * 0 < y' < H (the bounds mask 0 < x' <= W, then the clip that gives x' = W zero weight).  A non-finite x' or y'
 * contributes nothing and does not poison the sample.  The reference instead zeroes the masked events and piles them
 * at (0, 0) as events with p = 0 and t = 0 (objectives.py:543-545).  tau and the images are those of
 * evk_flow_timestamp_objective_f32: per polarity s (p > 0 / p <= 0; a NaN p is dropped), on the (H+1)x(W+1) canvas,
 *   T_s = S_s / C_s,  S_s = sum tau k,  C_s = 1 + sum k,   f_b = sum gaussian_filter(T_+, blur_sigma)^2 + sum (...T_-...)^2
 * the negation of zhu_timestamp_objective.evaluate_function.  blur_sigma follows the blur-sigma rule of the other
 * entries (0 or less: no blur; NaN: EVK_E_ARG; a radius over 64: EVK_E_UNSUPPORTED), checked before any CUDA call.
 *   x, y, t_rel, tau, p : n_events floats;  offsets: batch+1 int64 on the device
 *   f_out: batch doubles;  ts_out, cnt_out: [batch][2][H+1][W+1] floats (T and C, polarity 0 positive), which the
 *   backward takes as ts_img, cnt_img.  0 <= batch <= 32767.
 * evk_motion_timestamp_objective_grad_f32 writes grad_params [batch][K] doubles = grad_f[b] df_b/dparams[b], the exact
 * derivative of the f above with the floor and keep decisions held (grad_f: batch floats on the device): with
 * U_s = G(2 grad_f[b] G_s), A_s = U_s / C_s and B_s = -U_s T_s / C_s, per contributing event of polarity s and each of
 * its four taps q = tau A_s + B_s,
 *   df/dx' = (1-dy)(q01-q00) + dy(q11-q10),  df/dy' = (1-dx)(q10-q00) + dx(q11-q01),
 *   df/dparams_k += df/dx' dx'/dparams_k + df/dy' dy'/dparams_k.
 * workspace: evk_motion_timestamp_objective_workspace_bytes(batch, H, W) bytes, 256-byte aligned, for either call; 0 for
 * arguments the entries reject (the canvas of every batched entry is at most 2^30 pixels (H+1)(W+1)).
 * Neither call synchronises, and both launch the same kernels whatever the batch. */
size_t evk_motion_timestamp_objective_workspace_bytes(int batch, int H, int W);
int evk_motion_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                       const float *p, const int64_t *offsets, int batch, int64_t n_events, int warp,
                                       const double *params, int K, double cx, double cy, int H, int W, double blur_sigma,
                                       double *f_out, float *ts_out, float *cnt_out, void *workspace,
                                       size_t workspace_bytes, void *stream);
int evk_motion_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                            const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                            int warp, const double *params, int K, double cx, double cy, int H, int W,
                                            double blur_sigma, const float *ts_img, const float *cnt_img,
                                            const float *grad_f, double *grad_params, void *workspace,
                                            size_t workspace_bytes, void *stream);

/* Many parameter vectors per sample in one pass over the events, for the average-timestamp loss: the sample points of a
 * grid search per window or the step lengths of a batched line search.  f_out[b][j] is exactly the f_b of
 * evk_motion_timestamp_objective_f32 with params[b] = cand[b][j]: the same warp, keep rule, NaN-polarity rule, stamps
 * tau and blur, the same argument checks and the blur-sigma rule for blur_sigma (0 or less: no blur; NaN: EVK_E_ARG; a
 * radius over 64: EVK_E_UNSUPPORTED), all checked before any CUDA call.  Forward only: no image out, no gradient.
 *   cand : [batch][n_cand][K] doubles in DEVICE memory, 1 <= n_cand <= 32, batch * n_cand <= 32767
 *   f_out: [batch][n_cand] doubles
 * Every event is read once and splatted under each of its sample's n_cand candidates.
 * workspace: evk_motion_timestamp_candidates_workspace_bytes(batch, n_cand, H, W) bytes (about 96 bytes per canvas pixel
 * and candidate), 256-byte aligned; the query returns 0 for arguments the entry rejects.
 * The call does not synchronise and launches the same kernels whatever batch and n_cand. */
size_t evk_motion_timestamp_candidates_workspace_bytes(int batch, int n_cand, int H, int W);
int evk_motion_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                        const float *p, const int64_t *offsets, int batch, int64_t n_events, int warp,
                                        const double *cand, int n_cand, int K, double cx, double cy, int H, int W,
                                        double blur_sigma, double *f_out, void *workspace, size_t workspace_bytes,
                                        void *stream);

/* Camera motion with known depth for the average-timestamp loss: the three entries above with inv_depth (n_events
 * floats on the device) inserted right after p, for EVK_WARP_CAMERA_MOTION only, with K = 8 and the warp, keep rules,
 * derivatives and identities of evk_cmax_motion_depth_objective_f32.  Everything else is the twin's. */
size_t evk_motion_timestamp_depth_objective_workspace_bytes(int batch, int H, int W);
int evk_motion_timestamp_depth_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                             const float *p, const float *inv_depth, const int64_t *offsets, int batch,
                                             int64_t n_events, int warp, const double *params, int K, double cx,
                                             double cy, int H, int W, double blur_sigma, double *f_out, float *ts_out,
                                             float *cnt_out, void *workspace, size_t workspace_bytes, void *stream);
int evk_motion_timestamp_depth_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                                  const float *p, const float *inv_depth, const int64_t *offsets,
                                                  int batch, int64_t n_events, int warp, const double *params, int K,
                                                  double cx, double cy, int H, int W, double blur_sigma,
                                                  const float *ts_img, const float *cnt_img, const float *grad_f,
                                                  double *grad_params, void *workspace, size_t workspace_bytes,
                                                  void *stream);
size_t evk_motion_timestamp_depth_candidates_workspace_bytes(int batch, int n_cand, int H, int W);
int evk_motion_timestamp_depth_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                              const float *p, const float *inv_depth, const int64_t *offsets,
                                              int batch, int64_t n_events, int warp, const double *cand, int n_cand,
                                              int K, double cx, double cy, int H, int W, double blur_sigma,
                                              double *f_out, void *workspace, size_t workspace_bytes, void *stream);

/* The dense-flow average-timestamp loss with the flow of every sample given on a coarse grid of nodes: the node grid,
 * its interpolation and limits of evk_cmax_grid_flow_objective_f32 (grid_flow: [batch][2][gh][gw] f32 on the device,
 * 2 <= gh <= H, 2 <= gw <= W, gh * gw <= 4096; align_corners nodes, f32 ratios rx, ry, zero for node taps outside the
 * grid), then everything of evk_flow_timestamp_objective_f32 at the interpolated flow: x' = x + u t_rel,
 * y' = y + v t_rel in f32, kept iff 0 <= x' < W and 0 <= y' < H, a NaN f for a sample with a non-finite x' or y', a
 * NaN p dropped, the T and C images per polarity, the blur and f_b = sum G(T_+)^2 + sum G(T_-)^2.  For events at
 * integer pixels inside the sensor, f equals the dense-flow f of the flow that bilinear upsampling with align_corners
 * makes of the nodes, to f32 rounding; at gh = H, gw = W the grid is the dense flow.
 *   f_out: batch doubles;  ts_out, cnt_out: [batch][2][H+1][W+1] floats, which the backward takes as ts_img, cnt_img.
 *   0 <= batch <= 32767.
 * evk_grid_flow_timestamp_objective_grad_f32 writes grad_grid [batch][2][gh][gw] floats = grad_f[b] df_b/dgrid_flow[b]:
 * df/dx' and df/dy' of evk_flow_timestamp_objective_grad_f32, times t_rel, spread over the event's four node taps with
 * their bilinear weights, summed per CTA in shared memory and across CTAs in f64, then rounded to f32.
 * workspace: evk_grid_flow_timestamp_objective_workspace_bytes(batch, gh, gw, H, W) bytes, 256-byte aligned, for
 * either call; 0 for arguments the entries reject.  All limits and the blur-sigma rule are checked before any CUDA
 * call.  Neither call synchronises, and both launch the same kernels whatever the batch. */
size_t evk_grid_flow_timestamp_objective_workspace_bytes(int batch, int gh, int gw, int H, int W);
int evk_grid_flow_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                          const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                          const float *grid_flow, int gh, int gw, int H, int W, double blur_sigma,
                                          double *f_out, float *ts_out, float *cnt_out, void *workspace,
                                          size_t workspace_bytes, void *stream);
int evk_grid_flow_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                               const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                               const float *grid_flow, int gh, int gw, int H, int W, double blur_sigma,
                                               const float *ts_img, const float *cnt_img, const float *grad_f,
                                               float *grad_grid, void *workspace, size_t workspace_bytes, void *stream);

/* Many node grids per sample in one pass over the events, for the grid-flow average-timestamp loss (a batched line
 * search of a grid-flow fit): f_out[b][j] is exactly the f_b of evk_grid_flow_timestamp_objective_f32 with
 * grid_flow[b] = cand[b][j].  A non-finite warped position makes only that candidate's f NaN.
 *   cand : [batch][n_cand][2][gh][gw] floats on the device, 1 <= n_cand <= 32, n_cand * gh * gw <= 12288,
 *          batch * n_cand <= 32767
 *   f_out: [batch][n_cand] doubles
 * Every event is read once; its node cell and weights are computed once and used for every candidate.  All limits are
 * checked before any CUDA call.  Forward only.  workspace: evk_grid_flow_timestamp_candidates_workspace_bytes(batch,
 * n_cand, gh, gw, H, W) bytes (about 96 bytes per canvas pixel and candidate), 256-byte aligned; 0 for arguments the
 * entry rejects.  The call does not synchronise and launches the same kernels whatever batch and n_cand. */
size_t evk_grid_flow_timestamp_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W);
int evk_grid_flow_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                           const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                           const float *cand, int n_cand, int gh, int gw, int H, int W,
                                           double blur_sigma, double *f_out, void *workspace, size_t workspace_bytes,
                                           void *stream);

/* Depth from a known camera motion with the average-timestamp loss: the inverse depth of every event interpolated from
 * a gh x gw grid of nodes of its sample, exactly as in evk_cmax_depth_grid_objective_f32 (motion rows, principal point,
 * node layout, f32 weights, zero outside taps, rotation once per pass), then the loss of
 * evk_motion_timestamp_depth_objective_f32 at that rho.
 *   motion        : [batch][8] doubles on the device, rows (wx, wy, wz, vx, vy, vz, fx, fy) (data: no gradient)
 *   inv_depth_grid: [batch][gh][gw] f32 on the device, 2 <= gh <= H, 2 <= gw <= W, gh * gw <= 4096
 *   tau           : the normalised stamps of evk_motion_timestamp_objective_f32
 * Keep rules: an event with a negative or non-finite rho, with Pz <= 0 or a non-finite Pz, or outside the bounds mask
 * (0 < x' <= W, 0 < y' <= H) contributes nothing, with weight 1, and so does an event with a NaN p; a non-finite warp
 * flags no sample, so f is never NaN from the events.  The T and C images per polarity, the blur and
 * f_b = sum G(T_+)^2 + sum G(T_-)^2 are evk_motion_timestamp_objective_f32's.  Blur sigma: <= 0 blurs nothing, a
 * NaN is rejected (EVK_E_ARG) and a sigma whose radius round(4 sigma) exceeds 64 is EVK_E_UNSUPPORTED.
 *   f_out: batch doubles;  ts_out, cnt_out: [batch][2][H+1][W+1] floats, which the backward takes as ts_img, cnt_img.
 *   0 <= batch <= 32767.
 * evk_depth_grid_timestamp_objective_grad_f32 writes grad_grid [batch][gh][gw] floats = grad_f[b] df_b/dinv_depth_grid[b]:
 * per contributing event df/dx' and df/dy' of evk_motion_timestamp_objective_grad_f32 times
 *   dx'/drho = d fx iz (vx - X vz),  dy'/drho = d fy iz (vy - Y vz)   (d = t_rel)
 * spread over the event's four node taps with their bilinear weights, summed per CTA in shared memory and across CTAs
 * in f64, then rounded to f32.
 * Identities: at gh = H, gw = W with events at integer pixels rho is the node and f is
 * evk_motion_timestamp_depth_objective_f32's with that rho; for a constant grid c, f is that loss at rho = c to f32
 * rounding (the four f32 node weights need not sum to exactly 1); at v = 0 f is EVK_WARP_CAMERA_ROTATION's timestamp
 * loss, up to the order in which the f32 image sums add the taps, and the gradient is exactly zero (dx'/drho and
 * dy'/drho are exact zeros, so no node term is formed).
 * workspace: evk_depth_grid_timestamp_objective_workspace_bytes(batch, gh, gw, H, W) bytes (what the grid flow's
 * timestamp query returns), 256-byte aligned, for either call; 0 for arguments the entries reject.  All limits and the
 * blur-sigma rule are checked before any CUDA call.  Neither call synchronises, and both launch the same kernels
 * whatever the batch. */
size_t evk_depth_grid_timestamp_objective_workspace_bytes(int batch, int gh, int gw, int H, int W);
int evk_depth_grid_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                           const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                           const double *motion, double cx, double cy, const float *inv_depth_grid,
                                           int gh, int gw, int H, int W, double blur_sigma, double *f_out,
                                           float *ts_out, float *cnt_out, void *workspace, size_t workspace_bytes,
                                           void *stream);
int evk_depth_grid_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                                const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                                const double *motion, double cx, double cy,
                                                const float *inv_depth_grid, int gh, int gw, int H, int W,
                                                double blur_sigma, const float *ts_img, const float *cnt_img,
                                                const float *grad_f, float *grad_grid, void *workspace,
                                                size_t workspace_bytes, void *stream);

/* Many inverse-depth grids per sample in one pass over the events, for the depth-grid average-timestamp loss:
 * f_out[b][j] is exactly the f_b of evk_depth_grid_timestamp_objective_f32 with inv_depth_grid[b] = cand[b][j].
 *   cand : [batch][n_cand][gh][gw] floats on the device, 1 <= n_cand <= 32, n_cand * gh * gw <= 12288,
 *          batch * n_cand <= 32767
 *   f_out: [batch][n_cand] doubles
 * Every event is read once (20 bytes); its node cell, weights and rotation are computed once and used for every
 * candidate.  All limits are checked before any CUDA call.  Forward only.  workspace:
 * evk_depth_grid_timestamp_candidates_workspace_bytes(batch, n_cand, gh, gw, H, W) bytes, 256-byte aligned; 0 for
 * arguments the entry rejects.  The call does not synchronise and launches the same kernels whatever batch and
 * n_cand. */
size_t evk_depth_grid_timestamp_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W);
int evk_depth_grid_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                            const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                            const double *motion, double cx, double cy, const float *cand,
                                            int n_cand, int gh, int gw, int H, int W, double blur_sigma,
                                            double *f_out, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * RobustNorm (row f4): clamp a tensor between two of its order statistics and rescale it.  Replaces
 * RobustNorm.__call__ / .percentile, lib/data_loaders/data_augmentation.py:82-130 (two kthvalue sorts),
 * the step after the voxel grid in the loaders (base_dataset.py:471).
 *   k_low / k_top: 1-based ranks, k = 1 + round(.01 q (n-1)) computed by the caller (:100)
 *   out = x if both statistics are 0, else (clamp(x, t_min, t_max) - min(t_min, t_max)) / (t_max + 1e-6);
 *   NaNs rank above +inf (as in kthvalue), and any NaN in x makes every element of out NaN unless out = x
 *   t_min_max: optional 2 floats on the device receiving the two statistics.
 * --------------------------------------------------------------------------------------------- */
size_t evk_robust_norm_workspace_bytes(void);
int evk_robust_norm_f32(const float *x, int64_t n, int64_t k_low, int64_t k_top, float *out,
                        float *t_min_max, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Host-buffer pipeline: the same voxel build for events living in HOST memory (pinned memory
 * gives full PCIe bandwidth).  Events are streamed in chunks through a double-buffered device
 * staging area so the H2D copy of chunk k+1 overlaps the scatter of chunk k; the finished grid
 * is copied back to `out_host`.  Synchronous (returns when out_host is complete).
 * *oob_host receives the out-of-range event count.
 * With EVK_AUTO_SPAN the span is that of the whole stream, read from the host arrays before the first
 * chunk: t0 = t[0], dt = t[n-1] - t[0] in float32 (evk_voxel_host_f32), t_first = t[0], t_last = t[n-1]
 * in float64 (evk_voxel_host_packed_f32); the t0 / dt / t_first / t_last arguments are then ignored.
 * Every chunk is scattered with that one span.
 * --------------------------------------------------------------------------------------------- */
typedef struct evk_pipeline evk_pipeline_t;
int evk_pipeline_create(evk_pipeline_t **pipe, int64_t chunk_events);
void evk_pipeline_destroy(evk_pipeline_t *pipe);
int evk_voxel_host_f32(evk_pipeline_t *pipe, const float *x, const float *y, const float *t,
                       const float *p, int64_t n, float t0, float dt, int B, int H, int W,
                       unsigned flags, float *out_host, unsigned long long *oob_host);
/* the same for host arrays in the storage layout (see evk_voxel_packed_f32): 13 B/event over PCIe */
int evk_voxel_host_packed_f32(evk_pipeline_t *pipe, const int16_t *x, const int16_t *y, const double *t,
                              const uint8_t *p, int64_t n, double t_first, double t_last, int B, int H,
                              int W, unsigned flags, float *out_host, unsigned long long *oob_host);

/* ---------------------------------------------------------------------------------------------
 * 64-bit content hash of a HOST buffer (every byte enters; multi-threaded above 2 MiB, result independent
 * of the thread count).  The identity of an event set in the host-side cache of uploaded events: the
 * reference's objective is a pure function of the arrays it is handed at every call
 * (lib/contrast_max/objectives.py:211-236), so a cached device copy may only be reused when the host
 * arrays are byte-identical to the ones that were uploaded.  No device work.
 * --------------------------------------------------------------------------------------------- */
uint64_t evk_host_hash64(const void *data, size_t nbytes, uint64_t seed);
/* k buffers in one call (one pool of threads for all of them); out[a] = hash of buffer a under a seed derived from
 * `seed` and a, so equal contents at different positions hash differently. */
void evk_host_hash64_multi(const void *const *ptrs, const size_t *nbytes, int k, uint64_t seed, uint64_t *out);

/* The staging copy of the host pipeline, for callers that fill their own pinned buffers: k host arrays of `nbytes`
 * each, dst[a] <- src[a], in 1 MiB blocks on 8 threads (EVK_HOST_COPY_THREADS) of the library's persistent worker
 * pool (half of the CPUs the process may run on, at most 32; EVK_HOST_THREADS) with non-temporal stores (the destination
 * is read next by the DMA engine, not by the CPU; EVK_HOST_COPY_STREAM=0 -> memcpy).  evk_voxel_host_f32 uses it for ordinary pageable sources -- what the
 * reference's loaders produce (lib/data_loaders/base_dataset.py:446-453).  No device work. */
void evk_host_copy(void *const *dst, const void *const *src, int k, size_t nbytes);
/* Upload k host arrays (nbytes[a] each) into device buffers the caller allocated -- the event set of a
 * contrast-maximisation run (the reference hands numpy arrays to every objective call, lib/contrast_max/objectives.py:211),
 * numpy inputs of the image functions.  Pageable sources go through the pipeline's pinned bounce slots, filled by the
 * worker pool while the previous pieces are on the wire; pinned sources are copied directly.  Synchronous: the data is on
 * the device when it returns.  A pipeline serves one call at a time. */
int evk_host_upload(evk_pipeline_t *pipe, void *const *dst_dev, const void *const *src_host, int k, const size_t *nbytes);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* EVK_H_ */
