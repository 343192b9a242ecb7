// evk_cmax.cu -- fused contrast-maximisation evaluation on H100:
//   warp -> bounds mask -> bilinear IWE (+ Jacobian-weighted derivative images) -> Gaussian
//   blur -> variance objective and its analytic gradient, one pass over the events.
//
// Semantics (reference):
//   linvel_warp.warp              lib/contrast_max/warps.py:51-61        (f64)
//   events_bounds_mask            lib/util/event_util.py:26-27           (f64)
//   get_iwe                       lib/contrast_max/objectives.py:184-192
//   events_to_image_drv           lib/representations/image.py:179-217   (f64 -> f32 cast, splat)
//   interpolate_to_derivative_img lib/representations/image.py:131-135
//   variance_objective            lib/contrast_max/objectives.py:231-236, 251-264
//   warp_events_flow_torch + IWE  lib/transforms/optic_flow.py:37-44, lib/visualization/draw_flow.py:18-21
//
// Design (DESIGN.md section 4):
//   * ONE pass over the events.  The accumulator is an array of 32-byte BLOCKS, one per pixel:
//     block (y,x) = {I_TL, I_TR, I_BL, I_BR, a, b, c, d} collects every event whose bilinear
//     footprint is anchored at (y,x) (each pixel therefore lives in four blocks; a gather kernel
//     folds them).  The 2x2 IWE footprint of an event is ONE red.global.add.v4.f32
//     (REDG.E.ADD.F32x4); the 8 derivative taps have only 4 free values (the taps of a derivative
//     image come in +/- pairs, image.py:131-135), so both derivative images are ONE more vector
//     reduction: 1 RED per event for f, 2 for f and g, instead of 4 / 12 scalar ones.  A scatter
//     kernel pays per RED lane-operation, whatever its width (scalar, v2, v4) and whether or not
//     lanes share a sector -- the count of reduction operations is what has to be minimised.  The accumulator (181*241*32 B = 1.4 MB
//     per replica, R <= 8 replicas against same-address serialisation) never leaves L2.
//   * ON-CHIP IWE (round 2, large event counts): the whole 181x241 image of warped events is 174 KB -- it
//     fits in ONE SM's shared memory.  cmax_onchip_kernel runs one 1024-thread CTA per SM, each with a
//     PRIVATE fixed-point image in shared memory; the four bilinear taps are native integer shared-memory
//     atomics (ATOMS.ADD: 4 per event hide under the HBM read of the events, while f32 shared atomics are
//     CAS loops and every L2 reduction is paid per event).  Fixed point = value * 2^22 in
//     a biased u32 cell; the RETURNING atomic tells the thread whether ITS add wrapped the 32-bit cell and
//     that thread carries +-2^10 out to the global accumulator, so the sum is exact integer arithmetic with
//     no overflow whatever the stream (per-tap quantisation 2^-23, below f32 rounding of the reference's
//     own accumulation).  Events with |p*mask| > 1 or non-finite weights take the global f32 path.  At
//     the end every CTA converts its image to f32 in place and adds it to a planar global image with TMA
//     bulk reductions (cp.reduce.async.bulk.global.shared::cta.add.f32, SASS UBLKRED) -- "finished tiles
//     leave through TMA".  The derivative images do not fit next to the IWE (3 x 174 KB), so with the
//     gradient their four free values per event remain ONE vector reduction to the L2 block accumulator.
//   * The reference blurs both derivative images and multiplies by the un-blurred IWE.  The
//     reflect-boundary Gaussian is self-adjoint, so  sum(2(I-mu) * G(D_k)) == sum(G(2(I-mu)) * D_k)
//     and G(2(I-mu)) = 2(G(I)-mu): ONE blur of ONE image (which f needs anyway) serves f and g.
//   * scipy blurs the (2,H,W) derivative stack along its length-2 axis as well
//     (objectives.py:253), mixing the two gradient components by [[a,b],[b,a]]; applied to the
//     two scalars at the end (host supplies a,b).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "evk_common.cuh"

namespace evk {

constexpr int kMaxRadius = 64;
constexpr int kMaxReplicas = 8;
constexpr int kMaxCandidates = 32;  // parameter points per batched evaluation
constexpr int kBlockFloats = 8;   // one 32-byte block (= one L2 sector) per pixel: {I_TL, I_TR, I_BL, I_BR, a, b, c, d}

struct BlurTaps {
    int r;
    double w[kMaxRadius + 1];  // w[k] = weight at distance k (symmetric)
};

// Parameters of the rotation / 4-DoF motion models (host order of evk_cmax_warp_objective_*):
//   rotation  {cx, cy, omega}                  xyztheta  {hx, hy, hz, theta, cx, cy}
// The batched passes hold ModelOf<WARP> (below), which is this block for every model of up to 4 parameters.
template <int N>
struct ModelParams {
    double m[N];
};
using WarpModel = ModelParams<6>;

struct CmaxArgs {
    const void *x, *y, *t, *p;
    int64_t n;
    double vx, vy, t_ref;  // linvel
    double p_scale;        // polarity multiplier (objectives.py:225 uses 100)
    const float *flow;     // dense flow [2][Hs][Ws]
    const float2 *flow_uv; // the same, interleaved {u,v} per pixel (built per call in the workspace)
    float flow_t0;
    int Hm, Wm;  // bounds-mask size (img_size)
    int Hc, Wc;  // canvas = sensor + 1
    int abs_polarity;
    int replicas;
    float *acc;  // [R][Hc*Wc][8]
    int vec16;      // on-chip path: all four event arrays are 16-byte aligned
    float *planar;  // on-chip path: planar f32 image [npix padded to 4] the CTAs' shared-memory images are reduced into
    unsigned long long *oob;
    WarpModel model;  // rotation / xyztheta
};

enum { WARP_LINVEL_F64 = 0, WARP_LINVEL_F32 = 1, WARP_FLOW_F32 = 2,
       WARP_ROTATION_F64 = 3, WARP_ROTATION_F32 = 4, WARP_XYZTHETA_F64 = 5, WARP_XYZTHETA_F32 = 6,
       WARP_AFFINE_F32 = 7, WARP_HOMOGRAPHY_F32 = 8, WARP_CAMERA_ROTATION_F32 = 9, WARP_CAMERA_MOTION_F32 = 10 };

__host__ __device__ constexpr bool is_model_warp(int w) { return w >= WARP_ROTATION_F64; }
__host__ __device__ constexpr bool is_rotation(int w) { return w == WARP_ROTATION_F64 || w == WARP_ROTATION_F32; }
__host__ __device__ constexpr bool is_linvel(int w) { return w == WARP_LINVEL_F64 || w == WARP_LINVEL_F32; }
__host__ __device__ constexpr bool is_planar(int w) { return w == WARP_AFFINE_F32 || w == WARP_HOMOGRAPHY_F32; }
// the camera motion's events carry their inverse depth (Event<WARP>, EventSource::rho)
__host__ __device__ constexpr bool has_depth(int w) { return w == WARP_CAMERA_MOTION_F32; }
__host__ __device__ constexpr bool is_camera(int w) { return w == WARP_CAMERA_ROTATION_F32 || has_depth(w); }
// the camera rotation's row is (wx, wy, wz, fx, fy): the angular velocity, then the focal lengths; the camera motion's
// is (wx, wy, wz, vx, vy, vz, fx, fy), the linear velocity between them
__host__ __device__ constexpr int model_dims(int w)
{
    return is_linvel(w) ? 2 : is_rotation(w) ? 3 : w == WARP_AFFINE_F32 ? 6 : w == WARP_HOMOGRAPHY_F32 ? 8 :
           w == WARP_CAMERA_ROTATION_F32 ? 5 : w == WARP_CAMERA_MOTION_F32 ? 8 : 4;
}
// length of the Jacobian rows model_taps fills (at least 4: the smaller models keep the rows they always had)
__host__ __device__ constexpr int jac_dims(int w) { return model_dims(w) > 4 ? model_dims(w) : 4; }

// The parameter block of a model as model_taps reads it: the K parameters, then the fixed centre (cx, cy) of xyztheta
// and the planar models (the principal point of the camera rotation).  At least 6 doubles (WarpModel, the block of the
// single-window entries and of every model of up to 4 parameters); the larger models take K + 2, so that the smaller
// models keep their registers and shared memory.
__host__ __device__ constexpr int model_slots(int w) { return model_dims(w) + 2 > 6 ? model_dims(w) + 2 : 6; }
template <int WARP>
using ModelOf = ModelParams<model_slots(WARP)>;

// bilinear splat of weight w (and derivative weight a) at (xf, yf) on the canvas:
// image.py:199-207 (IWE) and :131-135 (derivative images) with w1 = [a;0], w2 = [0;a].
// PAIR: two adjacent lanes carry the SAME event; lane parity `xt` picks the x tap (x0 or x0+1) and
// the lane issues the two row taps of that column.  The two lanes of a pair then write 32
// contiguous bytes (pixels x0, x0+1 of the interleaved accumulator) in the same instruction, which
// the LSU merges into one L2 request per row: half the L2 tag look-ups of the one-lane-per-event
// form (L2 tag look-ups are what limits the scatter).
struct Taps {
    int x0, x1, y0, y1;
    float wm;     // masked weight (|wm| <= 1 is the fast-path condition of the on-chip image)
    float dx, dy; // bilinear fractions (the gradient pass of the motion models gathers with them)
    float4 ti;    // IWE taps TL, TR, BL, BR
    float4 td;    // free values of the derivative taps: a = am*oy, b = am*dy, c = am*ox, d = am*dx
};

// The arithmetic of one bilinear splat (image.py:199-207, :131-135), shared by the two accumulator back ends.
// Returns false when the event contributes nothing (out of the canvas -> counted, or all-zero weights).
template <bool GRAD>
__device__ __forceinline__ bool splat_taps(const CmaxArgs &A, float xf, float yf, float w, float a, bool clip, unsigned &oob, Taps &T)
{
    const float clipx = (float)(A.Wc - 1), clipy = (float)(A.Hc - 1);
    float m2 = 1.0f;
    if (clip) m2 = (xf >= clipx ? 0.0f : 1.0f) * (yf >= clipy ? 0.0f : 1.0f);
    const float pxf = floorf(xf), pyf = floorf(yf);
    const float dx = __fsub_rn(xf, pxf), dy = __fsub_rn(yf, pyf);
    int upx, upy;
    if (!trunc_checked(__fmul_rn(pxf, m2), upx) || !trunc_checked(__fmul_rn(pyf, m2), upy) ||
        !wrap_int_index(upx, A.Wc, T.x0) || !wrap_int_index(upx + 1, A.Wc, T.x1) ||
        !wrap_int_index(upy, A.Hc, T.y0) || !wrap_int_index(upy + 1, A.Hc, T.y1)) { ++oob; return false; }
    const float wm = __fmul_rn(w, m2);
    const float am = GRAD ? __fmul_rn(a, wm) : 0.0f;  // jacobian * masked_ps (image.py:211-212)
    if (wm == 0.0f && am == 0.0f) return false;
    const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
    const float wl = __fmul_rn(wm, ox), wr = __fmul_rn(wm, dx);
    T.wm = wm;
    T.dx = dx; T.dy = dy;
    // tap order inside a block: TL (y0,x0), TR (y0,x1), BL (y1,x0), BR (y1,x1)
    T.ti = make_float4(__fmul_rn(wl, oy), __fmul_rn(wr, oy), __fmul_rn(wl, dy), __fmul_rn(wr, dy));
    // image.py:131-135 with w1 = [am;0], w2 = [0;am]:
    //   D0 taps = am*{-oy, +oy, -dy, +dy}   -> TL = -TR, BL = -BR : two free values a = am*oy, b = am*dy
    //   D1 taps = am*{-ox, -dx, +ox, +dx}   -> TL = -BL, TR = -BR : two free values c = am*ox, d = am*dx
    // (negation is exact and commutes with the sums, so accumulating a,b,c,d and restoring the
    // signs in the fold gives the same images) -> both derivative images are ONE vector reduction.
    T.td = make_float4(0.f, 0.f, 0.f, 0.f);
    if (GRAD) T.td = make_float4(__fmul_rn(am, oy), __fmul_rn(am, dy), __fmul_rn(am, ox), __fmul_rn(am, dx));
    return true;
}

// taps -> the global block accumulator.  WANT_I / WANT_D select the image taps and the derivative values.
template <bool WANT_I, bool WANT_D>
__device__ __forceinline__ void emit_global(const CmaxArgs &A, float *acc, const Taps &T)
{
    if (T.x1 == T.x0 + 1 && T.y1 == T.y0 + 1) {
        float *blk = acc + ((int64_t)T.y0 * A.Wc + T.x0) * kBlockFloats;
        if (WANT_I) red_add4(blk, T.ti);
        if (WANT_D) red_add4(blk + 4, T.td);
        return;
    }
    // wrapped footprint (negative coordinates, only reachable without the bounds mask): every tap
    // becomes the TL tap of its own pixel's block (TL of D0 is -a, TL of D1 is -c)
    const float vi[4] = {T.ti.x, T.ti.y, T.ti.z, T.ti.w};
    const float v0[4] = {-T.td.x, T.td.x, -T.td.y, T.td.y}, v1[4] = {-T.td.z, -T.td.w, T.td.z, T.td.w};
    const int ys[4] = {T.y0, T.y0, T.y1, T.y1}, xs[4] = {T.x0, T.x1, T.x0, T.x1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float *bk = acc + ((int64_t)ys[k] * A.Wc + xs[k]) * kBlockFloats;
        if (WANT_I && vi[k] != 0.0f) red_add(bk, vi[k]);
        if (WANT_D && v0[k] != 0.0f) red_add(bk + 4, -v0[k]);
        if (WANT_D && v1[k] != 0.0f) red_add(bk + 6, -v1[k]);
    }
}

// bilinear splat of weight w (and derivative weight a) at (xf, yf) on the canvas, L2 back end
template <bool GRAD>
__device__ __forceinline__ void splat(const CmaxArgs &A, float *acc, float xf, float yf, float w, float a,
                                      bool clip, unsigned &oob)
{
    Taps T;
    if (!splat_taps<GRAD>(A, xf, yf, w, a, clip, oob, T)) return;
    emit_global<true, GRAD>(A, acc, T);
}

// ---- on-chip back end: the IWE lives in the CTA's shared memory as biased fixed point ----------------
constexpr int kFixBits = 22;
constexpr float kFixScale = (float)(1 << kFixBits);
constexpr float kFixCarry = (float)(1u << (32 - kFixBits));   // value of one 2^32 wrap of a cell
constexpr unsigned kFixBias = 0x80000000u;

__device__ __forceinline__ unsigned atoms_add_ret(unsigned *cell, unsigned v)
{
    unsigned old;
    asm volatile("atom.relaxed.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"((unsigned)__cvta_generic_to_shared(cell)), "r"(v));
    return old;
}

// Did adding the signed increment q to the biased cell (old -> old + q mod 2^32) wrap the 32 bits?  A wrap flips the
// top bit TOWARDS the sign of q (carry: 1 -> 0 with q >= 0; borrow: 0 -> 1 with q < 0); the other top-bit flip is the
// true value crossing zero.  Bit 31 of the result is the answer; q == 0 never wraps.
__device__ __forceinline__ unsigned wrap_bit(unsigned old, unsigned q) { const unsigned nw = old + q; return (old ^ nw) & ~(nw ^ q); }

// The four taps of one event: four independent native shared-memory atomics, ONE rarely taken branch.
// A wrap of a cell is carried to the global accumulator (TL slot of the pixel's own block, which the fold
// adds to the pixel), so the total is exact integer arithmetic for any event count.
__device__ __forceinline__ void onchip_taps(unsigned *simg, float *acc, int p00, int p01, int p10, int p11, float4 ti)
{
    const unsigned q0 = (unsigned)__float2int_rn(__fmul_rn(ti.x, kFixScale));   // |tap| <= 1 -> |q| <= 2^22
    const unsigned q1 = (unsigned)__float2int_rn(__fmul_rn(ti.y, kFixScale));
    const unsigned q2 = (unsigned)__float2int_rn(__fmul_rn(ti.z, kFixScale));
    const unsigned q3 = (unsigned)__float2int_rn(__fmul_rn(ti.w, kFixScale));
    const unsigned o0 = atoms_add_ret(simg + p00, q0), o1 = atoms_add_ret(simg + p01, q1);
    const unsigned o2 = atoms_add_ret(simg + p10, q2), o3 = atoms_add_ret(simg + p11, q3);
    const unsigned w0 = wrap_bit(o0, q0), w1 = wrap_bit(o1, q1), w2 = wrap_bit(o2, q2), w3 = wrap_bit(o3, q3);
    if ((w0 | w1 | w2 | w3) >> 31) {
        if (w0 >> 31) red_add(acc + (int64_t)p00 * kBlockFloats, (int)q0 >= 0 ? kFixCarry : -kFixCarry);
        if (w1 >> 31) red_add(acc + (int64_t)p01 * kBlockFloats, (int)q1 >= 0 ? kFixCarry : -kFixCarry);
        if (w2 >> 31) red_add(acc + (int64_t)p10 * kBlockFloats, (int)q2 >= 0 ? kFixCarry : -kFixCarry);
        if (w3 >> 31) red_add(acc + (int64_t)p11 * kBlockFloats, (int)q3 >= 0 ? kFixCarry : -kFixCarry);
    }
}

template <bool GRAD>
__device__ __forceinline__ void splat_onchip(const CmaxArgs &A, float *acc, unsigned *simg, float xf, float yf, float w, float a,
                                             bool clip, unsigned &oob)
{
    Taps T;
    if (!splat_taps<GRAD>(A, xf, yf, w, a, clip, oob, T)) return;
    if (fabsf(T.wm) <= 1.0f) {      // false for NaN / inf as well
        const int r0 = T.y0 * A.Wc, r1 = T.y1 * A.Wc;
        onchip_taps(simg, acc, r0 + T.x0, r0 + T.x1, r1 + T.x0, r1 + T.x1, T.ti);
        if (GRAD) emit_global<false, true>(A, acc, T);
    } else {
        emit_global<true, GRAD>(A, acc, T);
    }
}

// One event's four components as loaded (f64 in parity mode, f32 otherwise).
template <int WARP> struct EvT { using type = float; };
template <> struct EvT<WARP_LINVEL_F64> { using type = double; };
template <> struct EvT<WARP_ROTATION_F64> { using type = double; };
template <> struct EvT<WARP_XYZTHETA_F64> { using type = double; };

template <int WARP>
struct Event {
    typename EvT<WARP>::type x, y, t, p;
};
// the camera motion's events also carry rho, the inverse depth of their scene point
template <>
struct Event<WARP_CAMERA_MOTION_F32> {
    float x, y, t, p, rho;
};

template <int WARP>
__device__ __forceinline__ Event<WARP> load_event(const CmaxArgs &A, int64_t i)
{
    using T = typename EvT<WARP>::type;
    Event<WARP> e;
    e.x = ld_stream((const T *)A.x + i);
    e.y = ld_stream((const T *)A.y + i);
    e.t = ld_stream((const T *)A.t + i);
    e.p = ld_stream((const T *)A.p + i);
    return e;
}

__device__ __forceinline__ void ld_vec16(const float *p, float (&v)[4])
{
    const float4 q = ld_stream4(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
}
__device__ __forceinline__ void ld_vec16(const double *p, double (&v)[2])
{
    const double2 q = ld_stream2(p);
    v[0] = q.x; v[1] = q.y;
}

// ---- rotation and 4-DoF motion models (contrast_max/warps.py defines them; the reference leaves them empty,
// lib/contrast_max/warps.py:63-83).  dt = t - t0 and the warp undoes the motion during dt:
//   rotation (cx, cy, omega):  a = omega dt, u = x - cx, v = y - cy
//     x' = cx + (cos(a) u + sin(a) v)          y' = cy + (cos(a) v - sin(a) u)
//     dx'/d(cx, cy, omega) = (1 - cos a, -sin a,  dt (cos(a) v - sin(a) u))
//     dy'/d(cx, cy, omega) = (sin a, 1 - cos a, -dt (cos(a) u + sin(a) v))
//   xyztheta (hx, hy, hz, theta) about the fixed centre (cx, cy):
//     x' = x - dt ((hx + hz u) - theta v)      y' = y - dt ((hy + hz v) + theta u)
//     dx'/d(hx, hy, hz, theta) = (-dt, 0, -dt u,  dt v)
//     dy'/d(hx, hy, hz, theta) = (0, -dt, -dt v, -dt u)
//   linvel (vx, vy), warps.py:51-61 (the batched motion objective; the single-window linvel entries keep their own
//   fused pass, cmax_event):  x' = x - dt vx,  y' = y - dt vy,  dx'/d(vx, vy) = (-dt, 0),  dy'/d(vx, vy) = (0, -dt)
//   affine (hx, hy, a11, a12, a21, a22) about the fixed centre (cx, cy), the batched passes only (f32):
//     sx = (hx + a11 u) + a12 v,  sy = (hy + a22 v) + a21 u,  x' = x - dt sx,  y' = y - dt sy
//     dx'/dp = (-dt, 0, -dt u, -dt v, 0, 0)      dy'/dp = (0, -dt, 0, 0, -dt u, -dt v)
//   homography (hx, hy, a11, a12, a21, a22, g1, g2): the first-order warp of the generator
//   [[a11, a12, hx], [a21, a22, hy], [g1, g2, 0]] on (u, v, 1), the batched passes only (f32):
//     nx = u - dt sx,  ny = v - dt sy,  q = dt ((g1 u) + (g2 v)),  w = 1 - q
//     x' = (x - dt sx) + nx q / w,  y' = (y - dt sy) + ny q / w        (= cx + nx / w, cy + ny / w)
//     dx'/d(hx .. a22) = affine's row / w,  dx'/d(g1, g2) = (nx dt u, nx dt v) / w^2  (y' likewise with ny)
//     An event with w <= 0 or a non-finite w has crossed the horizon and is not kept.  With g1 = g2 = 0, w is 1 and
//     the warp and Jacobian are affine's bit for bit; affine at (hx, hy, hz, -theta, theta, hz) is xyztheta's.
//   camera rotation (wx, wy, wz, fx, fy) with the principal point (cx, cy), exact in the rotation, the batched passes
//   only (f32): the camera's angular velocity in its own frame (x right, y down, z along the optical axis)
//     b = ((x - cx) / fx, (y - cy) / fy, 1),  theta = dt w,  phi = |theta|,  c = theta x b,  e = theta x c
//     P = exp([theta]x) b = (b + A c) + B e,  A = sin(phi) / phi,  B = (1 - cos(phi)) / phi^2
//     X = Px iz,  Y = Py iz,  iz = 1 / Pz,  x' = cx + fx X,  y' = cy + fy Y
//     A = r cos(phi/2) and B = r^2 / 2 with r = sin(phi/2) / (phi/2) (1 at phi = 0): no 0/0 and no 1 - cos.  The sine
//     and cosine of phi/2 come from sincospif((phi/2) (1/pi)), whose exact argument reduction needs no local memory.
//     An event with Pz <= 0 or a non-finite Pz has rotated behind the camera and is not kept.
//     dP/dw = -dt [P]x J_l,  J_l = A I + B [theta]x + C theta theta^T (the SO(3) left
//     Jacobian, C = (phi - sin(phi)) / phi^3, a series below kCamSeriesPhi), so
//       dx'/dw = -dt fx J_l^T (X Y, -(1 + X X), Y),     dy'/dw = -dt fy J_l^T (1 + Y Y, -X Y, -X)
//     and through b and the projection, with R e_x, R e_y the first two columns of exp([theta]x):
//       dx'/dfx = X - (bx iz) ((R e_x)_x - X (R e_x)_z),   dy'/dfx = -(bx iz) (fy / fx) ((R e_x)_y - Y (R e_x)_z)
//       dx'/dfy = -(by iz) (fx / fy) ((R e_y)_x - X (R e_y)_z),   dy'/dfy = Y - (by iz) ((R e_y)_y - Y (R e_y)_z)
//   camera motion (wx, wy, wz, vx, vy, vz, fx, fy) with the principal point (cx, cy) and the event's inverse depth rho,
//   the batched passes with depth only (f32): the camera rotation's branch with the translation added to P,
//     U = exp([theta]x) b (the rotation's P),  s = rho dt,  P = U + s v,  iz, X, Y, x', y' as above
//     exact for the camera pose (exp(dt [w]x), dt v) at t in the camera frame at t0.  An event with a negative or
//     non-finite rho is not kept, nor one with Pz <= 0 or a non-finite Pz.  At s v = 0 (rho = 0 or v = 0) the
//     translation adds an exact zero, so x', y' are the camera rotation's bit for bit.  With Q = U iz:
//       dx'/dw = -dt fx J_l^T (X Qy, -(Qz + X Qx), Qy),   dy'/dw = -dt fy J_l^T (Qz + Y Qy, -Y Qx, -Qx)
//       dx'/dv = s fx iz (1, 0, -X),   dy'/dv = s fy iz (0, 1, -Y),   d/dfx, d/dfy: the camera rotation's with this P
// in the order written (no FMA: the library builds with -fmad=false), f64 in parity mode, f32 in fast mode.
// THE one place that turns an event into its bilinear footprint for these models: warp, bounds mask
// (event_util.py:26-27), f64 -> f32 cast (image.py:180-183) and splat_taps -- the IWE pass and the gradient
// pass call it alike, so they see identical taps.  JAC: also the f32 Jacobian rows jx[k] = dx'/dp_k, jy[k].
__device__ __forceinline__ void sin_cos(double a, double *s, double *c) { sincos(a, s, c); }
__device__ __forceinline__ void sin_cos(float a, float *s, float *c) { sincosf(a, s, c); }
// below this rotation angle (rad) the camera rotation's C = (phi - sin phi) / phi^3 is its series: above it the f32
// difference keeps about 6 eps / phi^2 of relative accuracy (2e-6 here), below it the series' first omitted term,
// phi^8 / 39916800, is under 1e-10
constexpr float kCamSeriesPhi = 0.5f;

// The camera models' warp in two halves, which the camera branch of model_taps and the depth-grid passes share (f32, in
// the order written): cam_rotate is the rotation U = exp([theta]x) b of the event's bearing, which depends on neither
// rho nor v, and cam_project adds the translation s v (TRANSLATE) and projects.
struct CamRot {
    float fx, fy, cx, cy, bx, by, tx, ty, tz, p2, phi, sh, ch, A, B, Ux, Uy, Uz;
};
struct CamProj {
    float iz, X, Y, xw, yw;
};

__device__ __forceinline__ CamRot cam_rotate(float x, float y, float d, float wx, float wy, float wz, float fx, float fy,
                                             float cx, float cy)
{
    CamRot c;
    c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy;
    c.bx = (x - cx) / fx; c.by = (y - cy) / fy;
    c.tx = d * wx; c.ty = d * wy; c.tz = d * wz;
    const float tx = c.tx, ty = c.ty, tz = c.tz, bx = c.bx, by = c.by;
    c.p2 = (tx * tx + ty * ty) + tz * tz;
    c.phi = sqrtf(c.p2);
    const float half = 0.5f * c.phi;
    sincospif(half * (float)0.318309886183790671, &c.sh, &c.ch);   // sin, cos of phi / 2, reduced exactly: no local memory
    const float r = c.phi > 0.0f ? c.sh / half : 1.0f;
    c.A = r * c.ch; c.B = 0.5f * (r * r);
    const float c0 = ty - tz * by, c1 = tz * bx - tx, c2 = tx * by - ty * bx;
    const float e0 = ty * c2 - tz * c1, e1 = tz * c0 - tx * c2, e2 = tx * c1 - ty * c0;
    c.Ux = (bx + c.A * c0) + c.B * e0; c.Uy = (by + c.A * c1) + c.B * e1; c.Uz = (1.0f + c.A * c2) + c.B * e2;
    return c;
}

// false for Pz <= 0 or a non-finite Pz: behind the camera, not kept.  Without TRANSLATE, P = U (s, v unused).
template <bool TRANSLATE>
__device__ __forceinline__ bool cam_project(const CamRot &c, float s, float vx, float vy, float vz, CamProj &q)
{
    float Px = c.Ux, Py = c.Uy, Pz = c.Uz;
    if constexpr (TRANSLATE) {
        Px = c.Ux + s * vx;   // the translation s v: an exact zero added at s = 0 or v = 0
        Py = c.Uy + s * vy;
        Pz = c.Uz + s * vz;
    }
    if (!(Pz > 0.0f) || isinf(Pz)) return false;
    q.iz = 1.0f / Pz; q.X = Px * q.iz; q.Y = Py * q.iz;
    q.xw = c.cx + c.fx * q.X;
    q.yw = c.cy + c.fy * q.Y;
    return true;
}

// The f32 Jacobian rows of a camera model's warp at its rotation cr and projection cp: jx[k] = dx'/dp_k, jy[k] for the
// motion (wx, wy, wz, and with DEPTH vx, vy, vz at the translation scale s = rho d) and, in the two slots behind it
// (N - 2, N - 1), the focal lengths (fx, fy).  Shared by model_taps and the depth-grid joint backward, so both see the
// same rows bit for bit.
template <bool DEPTH, int N>
__device__ __forceinline__ void cam_jacobian(const CamRot &cr, const CamProj &cp, float s, float d, float (&jx)[N],
                                             float (&jy)[N])
{
    using R = float;
    constexpr int F = N - 2;
    const R fx = cr.fx, fy = cr.fy, bx = cr.bx, by = cr.by, tx = cr.tx, ty = cr.ty, tz = cr.tz, p2 = cr.p2;
    const R phi = cr.phi, sh = cr.sh, ch = cr.ch, A = cr.A, B = cr.B;
    const R iz = cp.iz, X = cp.X, Y = cp.Y;
    // (phi - sin phi) / phi^3 cancels in f32 for small phi: 1/6 - phi^2/120 + phi^4/5040 - phi^6/362880 there
    const R C = phi < kCamSeriesPhi
                    ? (R)(1.0 / 6) - p2 * ((R)(1.0 / 120) - p2 * ((R)(1.0 / 5040) - p2 * (R)(1.0 / 362880)))
                    : (phi - (R)2 * (sh * ch)) / (p2 * phi);
    // J_l^T w = A w - B (theta x w) + C theta (theta . w), scaled by s
    auto jlt = [&](R w0, R w1, R w2, R s, float (&j)[N]) {
        const R k0 = ty * w2 - tz * w1, k1 = tz * w0 - tx * w2, k2 = tx * w1 - ty * w0;
        const R q = C * ((tx * w0 + ty * w1) + tz * w2);
        j[0] = s * ((A * w0 - B * k0) + q * tx);
        j[1] = s * ((A * w1 - B * k1) + q * ty);
        j[2] = s * ((A * w2 - B * k2) + q * tz);
    };
    if constexpr (DEPTH) {
        const R Qx = cr.Ux * iz, Qy = cr.Uy * iz, Qz = cr.Uz * iz;
        jlt(X * Qy, -(Qz + X * Qx), Qy, -(d * fx), jx);
        jlt(Qz + Y * Qy, -(Y * Qx), -Qx, -(d * fy), jy);
        const R sx = (s * fx) * iz, sy = (s * fy) * iz;
        jx[3] = sx; jx[4] = 0.0f; jx[5] = -(sx * X);
        jy[3] = 0.0f; jy[4] = sy; jy[5] = -(sy * Y);
    } else {
        jlt(X * Y, -((R)1 + X * X), Y, -(d * fx), jx);
        jlt((R)1 + Y * Y, -(X * Y), -X, -(d * fy), jy);
    }
    const R rxx = (R)1 - B * (ty * ty + tz * tz), rxy = A * tz + B * (tx * ty), rxz = B * (tx * tz) - A * ty;
    const R ryx = B * (tx * ty) - A * tz, ryy = (R)1 - B * (tx * tx + tz * tz), ryz = A * tx + B * (ty * tz);
    const R ux = bx * iz, uy = by * iz;
    jx[F] = X - ux * (rxx - X * rxz);
    jy[F] = -(ux * (fy / fx)) * (rxy - Y * rxz);
    jx[F + 1] = -(uy * (fx / fy)) * (ryx - X * ryz);
    jy[F + 1] = Y - uy * (ryy - Y * ryz);
}

// event_util.py:26-27: keep iff 0 < x' <= Wm and 0 < y' <= Hm (NaN compares false -> kept), then the f32 splat taps
template <class R>
__device__ __forceinline__ bool model_keep_taps(const CmaxArgs &A, R xw, R yw, R p, unsigned &oob, Taps &T)
{
    const bool keep = !(xw <= (R)0 || xw > (R)A.Wm) && !(yw <= (R)0 || yw > (R)A.Hm);
    if (!keep) return false;
    return splat_taps<false>(A, (float)xw, (float)yw, (float)p, 0.0f, true, oob, T);
}

template <int WARP, bool JAC>
__device__ __forceinline__ bool model_taps(const CmaxArgs &A, const Event<WARP> &e, const ModelOf<WARP> &M, unsigned &oob,
                                           Taps &T, float (&jx)[jac_dims(WARP)], float (&jy)[jac_dims(WARP)])
{
    using R = typename EvT<WARP>::type;
    R p = e.p;
    if (A.p_scale != 1.0) p = p * (R)A.p_scale;
    if (A.abs_polarity) p = fabs(p);
    const R d = (sizeof(R) == 8) ? e.t - (R)A.t_ref : e.t;   // fast mode stores t - t_ref already
    R xw, yw;
    if (is_linvel(WARP)) {
        const R vx = (R)M.m[0], vy = (R)M.m[1];
        xw = e.x - d * vx;
        yw = e.y - d * vy;
        if (JAC) {
            jx[0] = (float)(-d); jx[1] = 0.0f;
            jy[0] = 0.0f; jy[1] = (float)(-d);
            jx[2] = jx[3] = jy[2] = jy[3] = 0.0f;
        }
    } else if (is_rotation(WARP)) {
        const R cx = (R)M.m[0], cy = (R)M.m[1], om = (R)M.m[2];
        R s, c;
        sin_cos(om * d, &s, &c);
        const R u = e.x - cx, v = e.y - cy;
        const R rx = c * u + s * v, ry = c * v - s * u;
        xw = cx + rx;
        yw = cy + ry;
        if (JAC) {
            jx[0] = (float)((R)1 - c); jx[1] = (float)(-s); jx[2] = (float)(d * ry);
            jy[0] = (float)s; jy[1] = (float)((R)1 - c); jy[2] = (float)(-(d * rx));
            jx[3] = jy[3] = 0.0f;
        }
    } else if constexpr (is_camera(WARP)) {
        constexpr int F = model_dims(WARP) - 2;   // the focal lengths' slots, behind the motion
        if constexpr (has_depth(WARP)) {
            if (!(e.rho >= (R)0) || isinf(e.rho)) return false;   // no depth: not kept, like an event off the canvas
        }
        const CamRot cr = cam_rotate(e.x, e.y, d, (R)M.m[0], (R)M.m[1], (R)M.m[2], (R)M.m[F], (R)M.m[F + 1], (R)M.m[F + 2],
                                     (R)M.m[F + 3]);
        R s = (R)0;
        if constexpr (has_depth(WARP)) s = e.rho * d;
        CamProj cp;
        // behind the camera: not kept, like an event off the canvas
        if (!cam_project<has_depth(WARP)>(cr, s, (R)M.m[3], (R)M.m[4], (R)M.m[5], cp)) return false;
        xw = cp.xw;
        yw = cp.yw;
        if (JAC) cam_jacobian<has_depth(WARP)>(cr, cp, s, d, jx, jy);
    } else if constexpr (is_planar(WARP)) {
        constexpr int K = model_dims(WARP);
        const R hx = (R)M.m[0], hy = (R)M.m[1], a11 = (R)M.m[2], a12 = (R)M.m[3], a21 = (R)M.m[4], a22 = (R)M.m[5];
        const R cx = (R)M.m[K], cy = (R)M.m[K + 1];
        const R u = e.x - cx, v = e.y - cy;
        const R sx = (hx + a11 * u) + a12 * v, sy = (hy + a22 * v) + a21 * u;
        const R mx = d * sx, my = d * sy;
        xw = e.x - mx;
        yw = e.y - my;
        const R du = d * u, dv = d * v;
        if constexpr (WARP == WARP_HOMOGRAPHY_F32) {
            const R g1 = (R)M.m[6], g2 = (R)M.m[7];
            const R nx = u - mx, ny = v - my;
            const R q = d * (g1 * u + g2 * v);
            const R w = (R)1 - q;
            if (!(w > (R)0) || isinf(w)) return false;   // past the horizon: not kept, like an event off the canvas
            xw = xw + nx * q / w;
            yw = yw + ny * q / w;
            if (JAC) {
                const R w2 = w * w;
                jx[0] = -d / w; jx[1] = 0.0f; jx[2] = -du / w; jx[3] = -dv / w; jx[4] = 0.0f; jx[5] = 0.0f;
                jy[0] = 0.0f; jy[1] = -d / w; jy[2] = 0.0f; jy[3] = 0.0f; jy[4] = -du / w; jy[5] = -dv / w;
                jx[6] = nx * du / w2; jx[7] = nx * dv / w2;
                jy[6] = ny * du / w2; jy[7] = ny * dv / w2;
            }
        } else if (JAC) {
            jx[0] = -d; jx[1] = 0.0f; jx[2] = -du; jx[3] = -dv; jx[4] = 0.0f; jx[5] = 0.0f;
            jy[0] = 0.0f; jy[1] = -d; jy[2] = 0.0f; jy[3] = 0.0f; jy[4] = -du; jy[5] = -dv;
        }
    } else {
        const R hx = (R)M.m[0], hy = (R)M.m[1], hz = (R)M.m[2], th = (R)M.m[3], cx = (R)M.m[4], cy = (R)M.m[5];
        const R u = e.x - cx, v = e.y - cy;
        xw = e.x - d * ((hx + hz * u) - th * v);
        yw = e.y - d * ((hy + hz * v) + th * u);
        if (JAC) {
            jx[0] = (float)(-d); jx[1] = 0.0f; jx[2] = (float)(-(d * u)); jx[3] = (float)(d * v);
            jy[0] = 0.0f; jy[1] = (float)(-d); jy[2] = (float)(-(d * v)); jy[3] = (float)(-(d * u));
        }
    }
    return model_keep_taps(A, xw, yw, p, oob, T);
}

// pass 1 of the motion models: the IWE only, through the same two accumulator back ends as linvel
template <int WARP, bool ONCHIP>
__device__ __forceinline__ void model_splat(const CmaxArgs &A, float *acc, const Event<WARP> &e, unsigned &oob, const WarpModel &M,
                                            unsigned *simg)
{
    Taps T;
    float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
    if (!model_taps<WARP, false>(A, e, M, oob, T, jx, jy)) return;
    if (ONCHIP && fabsf(T.wm) <= 1.0f) {
        const int r0 = T.y0 * A.Wc, r1 = T.y1 * A.Wc;
        onchip_taps(simg, acc, r0 + T.x0, r0 + T.x1, r1 + T.x0, r1 + T.x1, T.ti);
    } else {
        emit_global<true, false>(A, acc, T);
    }
}

// The flow at an event (optic_flow.py:37-44: normalise to [-1,1], grid_sample bilinear, zero padding, align_corners):
// u, v, and the four grid_sample taps (x0, y0) .. (x0+1, y0+1) with their weights nw, ne, sw, se, which the backward
// of the flow objective spreads its gradient over.  `sampled` is false for coordinates no tap can reach (u = v = 0).
struct FlowSample {
    int x0, y0;
    float nw, ne, sw, se;
    float u, v;
    bool sampled;
};

template <bool INTERLEAVED>
__device__ __forceinline__ FlowSample flow_sample(const float *flow, const float2 *uv, int H, int W, float xe, float ye)
{
    FlowSample s;
    const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
    const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(xe, wm1), 2.0f), 1.0f);
    const float gy = __fsub_rn(__fmul_rn(__fdiv_rn(ye, hm1), 2.0f), 1.0f);
    const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.0f), 2.0f), wm1);
    const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.0f), 2.0f), hm1);
    float u = 0.0f, v = 0.0f;
    s.sampled = fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f;
    s.x0 = s.y0 = 0;
    s.nw = s.ne = s.sw = s.se = 0.0f;
    if (s.sampled) {
        const float fx = floorf(ix), fy = floorf(iy);
        const int x0 = (int)fx, y0 = (int)fy;
        const float xs = fx + 1.0f, ys = fy + 1.0f;
        const float nw = __fmul_rn(__fsub_rn(xs, ix), __fsub_rn(ys, iy));
        const float ne = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(ys, iy));
        const float sw = __fmul_rn(__fsub_rn(xs, ix), __fsub_rn(iy, fy));
        const float se = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy));
        const float4 top = flow_row<INTERLEAVED>(flow, uv, H, W, y0, x0), bot = flow_row<INTERLEAVED>(flow, uv, H, W, y0 + 1, x0);
        u = __fadd_rn(u, __fmul_rn(top.x, nw)); v = __fadd_rn(v, __fmul_rn(top.y, nw));
        u = __fadd_rn(u, __fmul_rn(top.z, ne)); v = __fadd_rn(v, __fmul_rn(top.w, ne));
        u = __fadd_rn(u, __fmul_rn(bot.x, sw)); v = __fadd_rn(v, __fmul_rn(bot.y, sw));
        u = __fadd_rn(u, __fmul_rn(bot.z, se)); v = __fadd_rn(v, __fmul_rn(bot.w, se));
        s.x0 = x0; s.y0 = y0;
        s.nw = nw; s.ne = ne; s.sw = sw; s.se = se;
    }
    s.u = u; s.v = v;
    return s;
}

template <int WARP, bool GRAD, bool ONCHIP = false>
__device__ __forceinline__ void cmax_event(const CmaxArgs &A, float *acc, const Event<WARP> &e, unsigned &oob, double cvx,
                                           double cvy, unsigned *simg = nullptr)
{
    if constexpr (is_model_warp(WARP)) {
        model_splat<WARP, ONCHIP>(A, acc, e, oob, A.model, simg);   // IWE pass only: the gradient is cmax_grad_pass_kernel
        return;
    }
    if (WARP == WARP_LINVEL_F64) {
        const double x = e.x, y = e.y, t = e.t;
        double p = e.p;
        if (A.p_scale != 1.0) p = __dmul_rn(p, A.p_scale);
        if (A.abs_polarity) p = fabs(p);
        const double d = __dsub_rn(t, A.t_ref);
        const double xw = __dsub_rn(x, __dmul_rn(d, cvx));  // warps.py:52-54
        const double yw = __dsub_rn(y, __dmul_rn(d, cvy));
        // event_util.py:26-27: keep iff 0 < x' <= Wm and 0 < y' <= Hm (NaN compares false -> kept)
        const bool keep = !(xw <= 0.0 || xw > (double)A.Wm) && !(yw <= 0.0 || yw > (double)A.Hm);
        if (!keep) return;  // x,y,p,j all multiplied by 0: only exact zeros are added at (0,0)..(1,1)
        if (ONCHIP) splat_onchip<GRAD>(A, acc, simg, (float)xw, (float)yw, (float)p, (float)(-d), true, oob);
        else splat<GRAD>(A, acc, (float)xw, (float)yw, (float)p, (float)(-d), true, oob);  // image.py:180-183 casts
    } else if (WARP == WARP_LINVEL_F32) {
        const float x = e.x, y = e.y;
        const float d = e.t;  // already t - t_ref
        float p = e.p;
        if (A.p_scale != 1.0) p = __fmul_rn(p, (float)A.p_scale);
        if (A.abs_polarity) p = fabsf(p);
        const float vx = (float)cvx, vy = (float)cvy;
        const float xw = __fsub_rn(x, __fmul_rn(d, vx)), yw = __fsub_rn(y, __fmul_rn(d, vy));
        const bool keep = !(xw <= 0.0f || xw > (float)A.Wm) && !(yw <= 0.0f || yw > (float)A.Hm);
        if (!keep) return;
        if (ONCHIP) splat_onchip<GRAD>(A, acc, simg, xw, yw, p, -d, true, oob);
        else splat<GRAD>(A, acc, xw, yw, p, -d, true, oob);
    } else {
        // optic_flow.py:37-44 then events_to_image_torch(..., interpolation='bilinear') defaults
        const float xe = e.x, ye = e.y, te = e.t;
        float p = e.p;
        if (A.abs_polarity) p = fabsf(p);
        const FlowSample s = flow_sample<true>(A.flow, A.flow_uv, A.Hc - 1, A.Wc - 1, xe, ye);
        const float u = s.u, v = s.v;
        const float d = __fsub_rn(te, A.flow_t0);
        if (ONCHIP) splat_onchip<false>(A, acc, simg, __fadd_rn(xe, __fmul_rn(u, d)), __fadd_rn(ye, __fmul_rn(v, d)), p, 0.0f, true, oob);
        else splat<false>(A, acc, __fadd_rn(xe, __fmul_rn(u, d)), __fadd_rn(ye, __fmul_rn(v, d)), p, 0.0f, true, oob);
    }
}

// The event pass.  Memory-level parallelism matters as much as the reductions here: each thread
// first issues the loads of kBatch events (16 independent loads in flight), then warps and
// splats them (a load -> compute -> red chain per event is latency bound, whatever the number of
// reductions).
constexpr int kBatch = 4;

template <int WARP, bool GRAD>
__global__ void __launch_bounds__(256) cmax_scatter_kernel(const CmaxArgs A)
{
    unsigned oob = 0;
    float *acc = A.acc + (int64_t)(blockIdx.x % A.replicas) * A.Hc * A.Wc * kBlockFloats;
    const int64_t stride = (int64_t)gridDim.x * 256;
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    for (; i + (kBatch - 1) * stride < A.n; i += kBatch * stride) {
        Event<WARP> ev[kBatch];
#pragma unroll
        for (int k = 0; k < kBatch; ++k) ev[k] = load_event<WARP>(A, i + k * stride);
#pragma unroll
        for (int k = 0; k < kBatch; ++k) cmax_event<WARP, GRAD>(A, acc, ev[k], oob, A.vx, A.vy);
    }
    for (; i < A.n; i += stride) cmax_event<WARP, GRAD>(A, acc, load_event<WARP>(A, i), oob, A.vx, A.vy);
    flush_oob(A.oob, oob);
}

// The on-chip event pass: one persistent 1024-thread CTA per SM, private fixed-point IWE in shared memory.
constexpr int kOnchipThreads = 1024;
constexpr int kBulkFloats = 4096;   // 16 KB per TMA bulk reduction

template <int WARP, bool GRAD>
__global__ void __launch_bounds__(kOnchipThreads, 1) cmax_onchip_kernel(const CmaxArgs A)
{
    extern __shared__ __align__(128) unsigned simg[];   // [npad] biased fixed point, then f32 in place
    const int npix = A.Hc * A.Wc, npad = (npix + 3) & ~3;
    for (int i = threadIdx.x; i < npad; i += kOnchipThreads) simg[i] = kFixBias;
    __syncthreads();
    unsigned oob = 0;
    // derivative reductions and carries go to the L2 block accumulator (replicas against same-address serialisation)
    float *acc = A.acc + (int64_t)(blockIdx.x % A.replicas) * A.Hc * A.Wc * kBlockFloats;
    const int64_t stride = (int64_t)gridDim.x * kOnchipThreads;
    int64_t i = (int64_t)blockIdx.x * kOnchipThreads + threadIdx.x;
    if (A.vec16) {
        // 16-byte loads: 4 f32 events / 2 f64 events per vector, two vectors of every array in flight per thread
        using T = typename EvT<WARP>::type;
        constexpr int EPV = 16 / (int)sizeof(T);
        const int64_t nv = A.n / EPV;
        const T *px = (const T *)A.x, *py = (const T *)A.y, *pt = (const T *)A.t, *pp = (const T *)A.p;
        for (int64_t v = i; v < nv; v += 2 * stride) {
            const bool two = v + stride < nv;
            const int64_t v2 = two ? v + stride : v;
            T ex[2][EPV], ey[2][EPV], et[2][EPV], ep[2][EPV];
            ld_vec16(px + v * EPV, ex[0]); ld_vec16(py + v * EPV, ey[0]); ld_vec16(pt + v * EPV, et[0]); ld_vec16(pp + v * EPV, ep[0]);
            ld_vec16(px + v2 * EPV, ex[1]); ld_vec16(py + v2 * EPV, ey[1]); ld_vec16(pt + v2 * EPV, et[1]); ld_vec16(pp + v2 * EPV, ep[1]);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h == 1 && !two) break;
#pragma unroll
                for (int k = 0; k < EPV; ++k) {
                    Event<WARP> e;
                    e.x = ex[h][k]; e.y = ey[h][k]; e.t = et[h][k]; e.p = ep[h][k];
                    cmax_event<WARP, GRAD, true>(A, acc, e, oob, A.vx, A.vy, simg);
                }
            }
        }
        for (int64_t j = nv * EPV + i; j < A.n; j += stride) cmax_event<WARP, GRAD, true>(A, acc, load_event<WARP>(A, j), oob, A.vx, A.vy, simg);
    } else {
        constexpr int kB = (sizeof(typename EvT<WARP>::type) == 8) ? 2 : 4;   // loads in flight per thread (64-register budget at 1024 threads)
        for (; i + (kB - 1) * stride < A.n; i += kB * stride) {
            Event<WARP> ev[kB];
#pragma unroll
            for (int k = 0; k < kB; ++k) ev[k] = load_event<WARP>(A, i + k * stride);
#pragma unroll
            for (int k = 0; k < kB; ++k) cmax_event<WARP, GRAD, true>(A, acc, ev[k], oob, A.vx, A.vy, simg);
        }
        for (; i < A.n; i += stride) cmax_event<WARP, GRAD, true>(A, acc, load_event<WARP>(A, i), oob, A.vx, A.vy, simg);
    }
    flush_oob(A.oob, oob);
    __syncthreads();
    // fixed point -> f32 in place (an int32 sum rounds to f32 once, like a float accumulator's final value)
    float *fimg = reinterpret_cast<float *>(simg);
    for (int j = threadIdx.x; j < npad; j += kOnchipThreads)
        fimg[j] = __fmul_rn((float)(int)(simg[j] - kFixBias), 1.0f / kFixScale);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA engine
    __syncthreads();
    // the finished image leaves through TMA: bulk add-reductions of 16 KB pieces into the planar global image
    if ((threadIdx.x & 31) == 0) {
        for (int c = threadIdx.x >> 5; c * kBulkFloats < npad; c += kOnchipThreads / 32) {
            const int off = c * kBulkFloats;
            const int cnt = (npad - off < kBulkFloats) ? (npad - off) : kBulkFloats;
            const unsigned src = (unsigned)__cvta_generic_to_shared(fimg + off);
            asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(
                             __cvta_generic_to_global(A.planar + off)), "r"(src), "r"(cnt * 4) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // shared memory must outlive the engine's reads
    }
}

// K candidate parameter points in ONE pass over the events (grid_search_initial evaluates 25 points per
// level, events_cmax.py:241-311): every event is loaded once and splatted into K accumulators.
struct Candidates {
    int n;
    double vx[kMaxCandidates], vy[kMaxCandidates];
};

template <int WARP, bool GRAD>
__global__ void __launch_bounds__(256) cmax_scatter_batch_kernel(const CmaxArgs A, const Candidates C)
{
    unsigned oob = 0;
    const int64_t acc_stride = (int64_t)A.Hc * A.Wc * kBlockFloats;
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < A.n; i += 2 * stride) {
        const Event<WARP> e0 = load_event<WARP>(A, i);
        const bool has1 = i + stride < A.n;
        const Event<WARP> e1 = has1 ? load_event<WARP>(A, i + stride) : e0;
        for (int k = 0; k < C.n; ++k) {
            float *acc = A.acc + k * acc_stride;
            cmax_event<WARP, GRAD>(A, acc, e0, oob, C.vx[k], C.vy[k]);
            if (has1) cmax_event<WARP, GRAD>(A, acc, e1, oob, C.vx[k], C.vy[k]);
        }
    }
    flush_oob(A.oob, oob);
}

// The same for the rotation / 4-DoF models: K parameter points per pass over the events, f only
struct ModelCandidates {
    int n;
    WarpModel m[kMaxCandidates];
};

template <int WARP>
__global__ void __launch_bounds__(256) cmax_model_batch_kernel(const CmaxArgs A, const ModelCandidates C)
{
    unsigned oob = 0;
    const int64_t acc_stride = (int64_t)A.Hc * A.Wc * kBlockFloats;
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < A.n; i += 2 * stride) {
        const Event<WARP> e0 = load_event<WARP>(A, i);
        const bool has1 = i + stride < A.n;
        const Event<WARP> e1 = has1 ? load_event<WARP>(A, i + stride) : e0;
        for (int k = 0; k < C.n; ++k) {
            float *acc = A.acc + k * acc_stride;
            model_splat<WARP, false>(A, acc, e0, oob, C.m[k], nullptr);
            if (has1) model_splat<WARP, false>(A, acc, e1, oob, C.m[k], nullptr);
        }
    }
    flush_oob(A.oob, oob);
}

// ---- pass 2 of the motion models: the gradient, GATHERED from one image instead of scattered into K --------
// Every objective's gradient is g_k = s * sum_pix C * G(D_k) with a per-pixel coefficient image C (2(I - mu) for the
// variance, 2I for sos, exp(G) for soe, ...) and D_k the derivative splat of image.py:131-135 with w1 = jx_k wm,
// w2 = jy_k wm.  G is self-adjoint, so g_k = s * sum_pix W D_k with W = G(C), and per event the four taps of D_k
// against W are
//   Sx = oy (W01 - W00) + dy (W11 - W10)      Sy = ox (W10 - W00) + dx (W11 - W01)      U_k += wm (jx_k Sx + jy_k Sy)
// One persistent CTA per SM holds W (f32, the 174 KB of a 181x241 canvas) in shared memory, recomputes each event's
// warp and footprint (model_taps, as pass 1), gathers four shared-memory values and sums K products per thread in
// f64; no reduction per event whatever K is.
constexpr int kGradThreads = 512;

// The slopes of the bilinear interpolant of four gathered values q00 (y0, x0), q01 (y0, x1), q10 (y1, x0), q11 (y1, x1)
// at the fractions (dx, dy), in the caller's type R (f32 in the flow passes, f64 in the model passes).
template <class R>
__device__ __forceinline__ void tap_slopes(R ox, R oy, R dx, R dy, R q00, R q01, R q10, R q11, R &sx, R &sy)
{
    sx = oy * (q01 - q00) + dy * (q11 - q10);
    sy = ox * (q10 - q00) + dx * (q11 - q01);
}

// CTA reduction of every thread's u[K] (THREADS threads): warp shuffles, the warp sums in shared memory, then one f64
// atomic per component and CTA into dst[K]
template <int K, int THREADS>
__device__ __forceinline__ void cta_add(const double (&u)[K], double *dst)
{
    __shared__ double part[THREADS / 32][K];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double v = u[k];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) part[wid][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        double s = 0.0;
        for (int w = 0; w < THREADS / 32; ++w) s += part[w][threadIdx.x];
        atomicAdd(dst + threadIdx.x, s);
    }
}

template <int WARP>
__global__ void __launch_bounds__(kGradThreads, 1) cmax_grad_pass_kernel(const CmaxArgs A, const float *__restrict__ W, double *U)
{
    constexpr int K = model_dims(WARP);
    extern __shared__ __align__(16) float sW[];
    const int npix = A.Hc * A.Wc;
    for (int j = threadIdx.x; j < npix; j += kGradThreads) sW[j] = W[j];
    __syncthreads();
    double u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = 0.0;
    unsigned oob = 0;   // counted by pass 1
    auto one = [&](const Event<WARP> &e) {
        Taps T;
        float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
        if (!model_taps<WARP, true>(A, e, A.model, oob, T, jx, jy)) return;
        const int r0 = T.y0 * A.Wc, r1 = T.y1 * A.Wc;
        const double w00 = sW[r0 + T.x0], w01 = sW[r0 + T.x1], w10 = sW[r1 + T.x0], w11 = sW[r1 + T.x1];
        const double dx = T.dx, dy = T.dy, ox = 1.0 - dx, oy = 1.0 - dy, wm = T.wm;
        double sx, sy;
        tap_slopes(ox, oy, dx, dy, w00, w01, w10, w11, sx, sy);
#pragma unroll
        for (int k = 0; k < K; ++k) u[k] += wm * ((double)jx[k] * sx + (double)jy[k] * sy);
    };
    const int64_t stride = (int64_t)gridDim.x * kGradThreads;
    int64_t i = (int64_t)blockIdx.x * kGradThreads + threadIdx.x;
    for (; i + 3 * stride < A.n; i += 4 * stride) {
        Event<WARP> ev[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) ev[k] = load_event<WARP>(A, i + k * stride);
#pragma unroll
        for (int k = 0; k < 4; ++k) one(ev[k]);
    }
    for (; i < A.n; i += stride) one(load_event<WARP>(A, i));
    cta_add<K, kGradThreads>(u, U);
}

// ---- image-space tail (43.6 K pixels; negligible next to the event pass) ------------------
// sums[]: 0 sum(I)  1 sum(G)  2 sum(G^2)  3 sum(G*D0)  4 sum(G*D1)  5 sum(D0)  6 sum(D1)
// block-wide sum of v (all 256 threads participate), one atomicAdd(double) per block
__device__ __forceinline__ void block_add(double v, double *dst)
{
    __shared__ double part[8];
    const int lt = threadIdx.y * blockDim.x + threadIdx.x;   // blocks are 256 threads, 1-D or 32x8
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // protect `part` against the previous call's readers
    if ((lt & 31) == 0) part[lt >> 5] = v;
    __syncthreads();
    if (lt == 0) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += part[w];
        atomicAdd(dst, s);
    }
}

// CTA-wide sum in a FIXED order (shuffle tree, then the 8 warp sums left to right); valid on thread 0
__device__ __forceinline__ double block_sum_ordered(double v)
{
    __shared__ double part2[8];
    const int lt = threadIdx.y * blockDim.x + threadIdx.x;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((lt & 31) == 0) part2[lt >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (lt == 0) for (int w = 0; w < 8; ++w) s += part2[w];
    return s;
}

// Blocks -> planar images.  Block (y,x) holds the 2x2 footprint anchored at (y,x) in tap order
// TL,TR,BL,BR, so pixel (y,x) collects TL of block (y,x), TR of (y,x-1), BL of (y-1,x) and BR of
// (y-1,x-1), over all replicas.
__global__ void __launch_bounds__(256) cmax_gather_kernel(const float *__restrict__ acc, const float *__restrict__ planar,
                                                          int replicas, int Hc, int Wc,
                                                          float *__restrict__ I, float *__restrict__ D0,
                                                          float *__restrict__ D1, float *__restrict__ iwe_out,
                                                          float *__restrict__ diwe_out, double *sums,
                                                          const unsigned long long *oob_in = nullptr, unsigned long long *oob_out = nullptr)
{
    const int npix = Hc * Wc;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (oob_out && i == 0) *oob_out = *oob_in;
    float a = 0.f, b = 0.f, c = 0.f;
    if (i < npix) {
        const int y = i / Wc, x = i - y * Wc;
        if (planar) a = planar[i];      // the on-chip images (cmax_onchip_kernel); the blocks then hold carries / slow-path taps only
        for (int r = 0; r < replicas; ++r) {
            const float *base = acc + (int64_t)r * npix * kBlockFloats;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int by = y - (k >> 1), bx = x - (k & 1);
                if (by < 0 || bx < 0) continue;
                const float *blk = base + ((int64_t)by * Wc + bx) * kBlockFloats;
                a += blk[k];
                // D0 block = {-a, +a, -b, +b}, D1 block = {-c, -d, +c, +d} (see splat)
                b += (k == 0) ? -blk[4] : (k == 1) ? blk[4] : (k == 2) ? -blk[5] : blk[5];
                c += (k == 0) ? -blk[6] : (k == 1) ? -blk[7] : (k == 2) ? blk[6] : blk[7];
            }
        }
        I[i] = a; D0[i] = b; D1[i] = c;
        if (iwe_out) iwe_out[i] = a;
        if (diwe_out) { diwe_out[i] = b; diwe_out[npix + i] = c; }
    }
    block_add((double)a, sums + 0);
    block_add((double)b, sums + 5);
    block_add((double)c, sums + 6);
}

__device__ __forceinline__ int reflect_idx(int i, int n)
{
    if (n == 1) return 0;
    const int period = 2 * n;
    i %= period;
    if (i < 0) i += period;
    return i < n ? i : period - 1 - i;
}

// scipy applies axis 0 first and rounds the intermediate to f32.
// The image-space kernels below that take blockIdx.z treat it as the image index of a batch of images laid out one
// after the other (the flow objective's samples); every other launch has gridDim.z = 1.
__global__ void __launch_bounds__(256) cmax_blur_axis0_kernel(const float *__restrict__ I, float *__restrict__ tmp,
                                                              int Hc, int Wc, const BlurTaps taps)
{
    const size_t img = (size_t)blockIdx.z * Hc * Wc;
    I += img; tmp += img;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= Hc * Wc) return;
    const int y = i / Wc, x = i - y * Wc;
    double acc = (double)I[i] * taps.w[0];
    for (int k = 1; k <= taps.r; ++k)
        acc += ((double)I[reflect_idx(y - k, Hc) * Wc + x] + (double)I[reflect_idx(y + k, Hc) * Wc + x]) * taps.w[k];
    tmp[i] = (float)acc;
}

__global__ void __launch_bounds__(256) cmax_blur_axis1_sums_kernel(const float *__restrict__ tmp, const float *__restrict__ I,
                                                                   const float *__restrict__ D0, const float *__restrict__ D1,
                                                                   int Hc, int Wc, const BlurTaps taps, int do_blur,
                                                                   double *sums)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    double g = 0.0, d0 = 0.0, d1 = 0.0;
    if (i < Hc * Wc) {
        if (do_blur) {
            const int y = i / Wc, x = i - y * Wc;
            const float *row = tmp + y * Wc;
            double acc = (double)row[x] * taps.w[0];
            for (int k = 1; k <= taps.r; ++k)
                acc += ((double)row[reflect_idx(x - k, Wc)] + (double)row[reflect_idx(x + k, Wc)]) * taps.w[k];
            g = (double)(float)acc;
        } else {
            g = (double)I[i];
        }
        d0 = (double)D0[i]; d1 = (double)D1[i];
    }
    block_add(g, sums + 1);
    block_add(g * g, sums + 2);
    block_add(g * d0, sums + 3);
    block_add(g * d1, sums + 4);
}

// result[0]=f  [1]=g0  [2]=g1  [3]=sum(IWE)  [4]=oob events  [5]=var  [6],[7] un-mixed 2-D gradient
__global__ void cmax_final_kernel(const double *sums, const unsigned long long *oob, int npix, double mix_a,
                                  double mix_b, int want_grad, double *result)
{
    const double P = (double)npix;
    const double mean_g = sums[1] / P;
    const double var = sums[2] / P - mean_g * mean_g;
    const double mu = sums[0] / P;
    // g2d_k = -mean( 2 (G(I) - mu) D_k )   (adjoint form of objectives.py:256-262)
    const double g0 = -2.0 * (sums[3] - mu * sums[5]) / P;
    const double g1 = -2.0 * (sums[4] - mu * sums[6]) / P;
    result[0] = -var;
    result[1] = want_grad ? (mix_a * g0 + mix_b * g1) : 0.0;
    result[2] = want_grad ? (mix_b * g0 + mix_a * g1) : 0.0;
    result[3] = sums[0];
    result[4] = (double)(*oob);
    result[5] = var;
    result[6] = g0;
    result[7] = g1;
}

// ---- generic objective tail (the reference's other objective functions, objectives.py:266-596) ---
// All of them are  f = reduce(phi(G))  with G = G_sigma * IWE and  g_k = -c * sum( w * (G3d * dIWE)_k )
// for a per-pixel weight image w.  The reflect Gaussian is self-adjoint, so sum(w * G(D_k)) ==
// sum(G(w) * D_k): ONE more blur (of w) replaces the reference's blur of the (2,H,W) stack.
//   SOS / RMS (objectives.py:266-357)  f = -mean(G^2)          w = 2*IWE (un-blurred), c = 1/P
//   SOE  (:358-400)                    f = -mean(exp(G))       w = exp(G),             c = 1/P
//   MOA  (:401-430)                    f = -max(G)             no gradient
//   ISOA (:431-477)                    f = +#(G > thresh)      w = [G > thresh],       c = 1
//   SOSA (:478-523)                    f = -sum(exp(-p G))     w = -p exp(-p G),       c = 1
enum { OBJ_VARIANCE = 0, OBJ_SOS = 1, OBJ_SOE = 2, OBJ_MOA = 3, OBJ_ISOA = 4, OBJ_SOSA = 5 };

__device__ __forceinline__ unsigned encode_ordered(float f)
{
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float decode_ordered(unsigned u)
{
    const unsigned b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    float f; memcpy(&f, &b, 4); return f;
#endif
}

// axis-1 blur, result stored (the variance path only needs its sums and does not store it)
__global__ void __launch_bounds__(256) cmax_blur_axis1_store_kernel(const float *__restrict__ tmp, const float *__restrict__ I,
                                                                    int Hc, int Wc, const BlurTaps taps, int do_blur,
                                                                    float *__restrict__ G)
{
    const size_t img = (size_t)blockIdx.z * Hc * Wc;
    tmp += img; I += img; G += img;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= Hc * Wc) return;
    if (!do_blur) { G[i] = I[i]; return; }
    const int y = i / Wc, x = i - y * Wc;
    const float *row = tmp + y * Wc;
    double acc = (double)row[x] * taps.w[0];
    for (int k = 1; k <= taps.r; ++k)
        acc += ((double)row[reflect_idx(x - k, Wc)] + (double)row[reflect_idx(x + k, Wc)]) * taps.w[k];
    G[i] = (float)acc;
}

// gsums: 0 sum(G^2)  1 sum(exp(G))  2 sum(exp(-p G))  3 #(G > thresh)  4 sum(G)  5 sum(Gw*D0)  6 sum(Gw*D1)
__global__ void __launch_bounds__(256) cmax_obj_reduce_kernel(const float *__restrict__ G, const float *__restrict__ I, int npix,
                                                              int kind, double param, double *gsums, unsigned *gmax,
                                                              double *__restrict__ w)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    double g2 = 0.0, ge = 0.0, ga = 0.0, gc = 0.0, g1 = 0.0;
    float mx = -FLT_MAX;
    if (i < npix) {
        const float g = G[i];
        const double gd = (double)g;
        g1 = gd;
        g2 = (double)(g * g);                           // np.mean(iwe*iwe): f32 product
        if (kind == OBJ_SOE) ge = exp(gd);              // np.exp(iwe.astype(np.double))
        if (kind == OBJ_SOSA) ga = exp(-param * gd);    // np.exp(-p*iwe.astype(np.double))
        if (kind == OBJ_ISOA) gc = (g > (float)param) ? 1.0 : 0.0;
        mx = g;
        double wi = 0.0;
        if (kind == OBJ_SOS) wi = (double)(I[i] * 2.0f);                                  // (iwe*2.0), un-blurred IWE
        else if (kind == OBJ_SOE) wi = ge;
        else if (kind == OBJ_ISOA) wi = gc;
        else if (kind == OBJ_SOSA) wi = -param * exp((double)(float)(-param * gd));       // exp((-p*iwe).astype(double)): f32 product first
        w[i] = wi;
    }
    block_add(g2, gsums + 0);
    if (kind == OBJ_SOE) block_add(ge, gsums + 1);
    if (kind == OBJ_SOSA) block_add(ga, gsums + 2);
    if (kind == OBJ_ISOA) block_add(gc, gsums + 3);
    block_add(g1, gsums + 4);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) atomicMax(gmax, encode_ordered(mx));
}

__global__ void __launch_bounds__(256) cmax_blur_d_axis0_kernel(const double *__restrict__ w, double *__restrict__ wt, int Hc,
                                                                int Wc, const BlurTaps taps)
{
    const size_t img = (size_t)blockIdx.z * Hc * Wc;
    w += img; wt += img;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= Hc * Wc) return;
    const int y = i / Wc, x = i - y * Wc;
    double acc = w[i] * taps.w[0];
    for (int k = 1; k <= taps.r; ++k) acc += (w[reflect_idx(y - k, Hc) * Wc + x] + w[reflect_idx(y + k, Hc) * Wc + x]) * taps.w[k];
    wt[i] = acc;
}

__global__ void __launch_bounds__(256) cmax_blur_d_axis1_dot_kernel(const double *__restrict__ wt, const double *__restrict__ w,
                                                                    const float *__restrict__ D0, const float *__restrict__ D1,
                                                                    int Hc, int Wc, const BlurTaps taps, int do_blur, double *gsums)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    double a = 0.0, b = 0.0;
    if (i < Hc * Wc) {
        double gw;
        if (do_blur) {
            const int y = i / Wc, x = i - y * Wc;
            const double *row = wt + y * Wc;
            gw = row[x] * taps.w[0];
            for (int k = 1; k <= taps.r; ++k) gw += (row[reflect_idx(x - k, Wc)] + row[reflect_idx(x + k, Wc)]) * taps.w[k];
        } else {
            gw = w[i];
        }
        a = gw * (double)D0[i];
        b = gw * (double)D1[i];
    }
    block_add(a, gsums + 5);
    block_add(b, gsums + 6);
}

// result: [0]=f [1],[2]=g [3]=sum(IWE) [4]=oob events [5]=var or aux [6],[7]=un-mixed gradient
//         [8]=mean(G^2) [9]=sum(exp(-p G)) [10]=max(G) [11]=#(G>thresh)
__global__ void cmax_obj_final_kernel(int kind, const double *gsums, const unsigned *gmax, const double *sums,
                                      const unsigned long long *oob, int npix, double mix_a, double mix_b, int want_grad,
                                      double *result)
{
    const double P = (double)npix;
    double f = 0.0, c = 0.0;
    const double mx = (double)decode_ordered(*gmax);
    if (kind == OBJ_SOS) { f = -gsums[0] / P; c = 1.0 / P; }
    else if (kind == OBJ_SOE) { f = -gsums[1] / P; c = 1.0 / P; }
    else if (kind == OBJ_MOA) { f = -mx; c = 0.0; }
    else if (kind == OBJ_ISOA) { f = gsums[3]; c = 1.0; }
    else if (kind == OBJ_SOSA) { f = -gsums[2]; c = 1.0; }
    const double u0 = -c * gsums[5], u1 = -c * gsums[6];
    const bool grad = want_grad && kind != OBJ_MOA;
    result[0] = f;
    result[1] = grad ? (mix_a * u0 + mix_b * u1) : 0.0;
    result[2] = grad ? (mix_b * u0 + mix_a * u1) : 0.0;
    result[3] = sums[0];
    result[4] = (double)(*oob);
    result[5] = gsums[4] / P;
    result[6] = u0;
    result[7] = u1;
    result[8] = gsums[0] / P;
    result[9] = gsums[2];
    result[10] = mx;
    result[11] = gsums[3];
}

// ---- image-space tail of the motion models: f, the side values and the gradient pass's W = G(C) -----------
// gsums: 0 sum(G^2) (f32 products)  1 sum(exp(G))  2 sum(exp(-p G))  3 #(G > thresh)  4 sum(G)  5 sum(G^2) (f64 products)
// The variance's C = 2(I - mu) blurs to 2(G - mu); the mean drops out of the gradient (the four derivative taps of an
// event sum to zero), so W = 2G, written here.  The other objectives leave C in w (f64) for one more blur.
__global__ void __launch_bounds__(256) cmax_model_stats_kernel(const float *__restrict__ G, const float *__restrict__ I, int npix,
                                                               int kind, double param, double *gsums, unsigned *gmax,
                                                               double *__restrict__ w, float *__restrict__ Wvar)
{
    const size_t img = (size_t)blockIdx.z * npix;
    G += img; I += img; gsums += 8 * blockIdx.z; gmax += blockIdx.z;
    if (w) w += img;
    if (Wvar) Wvar += img;
    const int i = blockIdx.x * 256 + threadIdx.x;
    double g2 = 0.0, ge = 0.0, ga = 0.0, gc = 0.0, g1 = 0.0, gd2 = 0.0;
    float mx = -FLT_MAX;
    if (i < npix) {
        const float g = G[i];
        const double gd = (double)g;
        g1 = gd;
        gd2 = gd * gd;
        g2 = (double)(g * g);
        if (kind == OBJ_SOE) ge = exp(gd);
        if (kind == OBJ_SOSA) ga = exp(-param * gd);
        if (kind == OBJ_ISOA) gc = (g > (float)param) ? 1.0 : 0.0;
        mx = g;
        if (kind == OBJ_VARIANCE) {
            if (Wvar) Wvar[i] = 2.0f * g;
        } else if (w) {
            double wi = 0.0;
            if (kind == OBJ_SOS) wi = (double)(I[i] * 2.0f);
            else if (kind == OBJ_SOE) wi = ge;
            else if (kind == OBJ_ISOA) wi = gc;
            else if (kind == OBJ_SOSA) wi = -param * exp((double)(float)(-param * gd));
            w[i] = wi;
        }
    }
    block_add(g2, gsums + 0);
    if (kind == OBJ_SOE) block_add(ge, gsums + 1);
    if (kind == OBJ_SOSA) block_add(ga, gsums + 2);
    if (kind == OBJ_ISOA) block_add(gc, gsums + 3);
    block_add(g1, gsums + 4);
    block_add(gd2, gsums + 5);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) atomicMax(gmax, encode_ordered(mx));
}

// W = G(w) along axis 1 (after cmax_blur_d_axis0_kernel), stored as f32 for the gradient pass
__global__ void __launch_bounds__(256) cmax_blur_d_axis1_store_kernel(const double *__restrict__ wt, const double *__restrict__ w,
                                                                      int Hc, int Wc, const BlurTaps taps, int do_blur,
                                                                      float *__restrict__ Wout)
{
    const size_t img = (size_t)blockIdx.z * Hc * Wc;
    wt += img; w += img; Wout += img;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= Hc * Wc) return;
    double gw;
    if (do_blur) {
        const int y = i / Wc, x = i - y * Wc;
        const double *row = wt + y * Wc;
        gw = row[x] * taps.w[0];
        for (int k = 1; k <= taps.r; ++k) gw += (row[reflect_idx(x - k, Wc)] + row[reflect_idx(x + k, Wc)]) * taps.w[k];
    } else {
        gw = w[i];
    }
    Wout[i] = (float)gw;
}

// result (16 doubles): [0] f  [1..4] g (zero past dims)  [5] sum(IWE)  [6] events outside the canvas
//                      [7] mean(G)  [8] mean(G^2)  [9] sum(exp(-p G))  [10] max(G)  [11] #(G > thresh)  [12..15] 0
__global__ void cmax_model_final_kernel(int kind, const double *gsums, const unsigned *gmax, const double *sums,
                                        const unsigned long long *oob, int npix, const double *U, int dims, int want_grad,
                                        double *result)
{
    const double P = (double)npix;
    const double mx = (double)decode_ordered(*gmax);
    double f = 0.0, c = 0.0;
    if (kind == OBJ_VARIANCE) { const double m = gsums[4] / P; f = -(gsums[5] / P - m * m); c = 1.0 / P; }
    else if (kind == OBJ_SOS) { f = -gsums[0] / P; c = 1.0 / P; }
    else if (kind == OBJ_SOE) { f = -gsums[1] / P; c = 1.0 / P; }
    else if (kind == OBJ_MOA) { f = -mx; c = 0.0; }
    else if (kind == OBJ_ISOA) { f = gsums[3]; c = 1.0; }
    else if (kind == OBJ_SOSA) { f = -gsums[2]; c = 1.0; }
    const bool grad = want_grad && kind != OBJ_MOA;
    result[0] = f;
    for (int k = 0; k < 4; ++k) result[1 + k] = (grad && k < dims) ? -c * U[k] : 0.0;
    result[5] = sums[0];
    result[6] = (double)(*oob);
    result[7] = gsums[4] / P;
    result[8] = gsums[0] / P;
    result[9] = gsums[2];
    result[10] = mx;
    result[11] = gsums[3];
    for (int k = 12; k < 16; ++k) result[k] = 0.0;
}

// ---- fused variance tail: gather + both blur axes + all sums + the final scalars in ONE launch ---
// One CTA = an 8x32 tile of pixels.  It gathers the tile plus a halo of `r` pixels (reflected at the image
// border, like scipy's mode='reflect') straight from the block accumulator into shared memory, blurs
// vertically then horizontally with the same f64-accumulate / f32-store rounding as the separate kernels,
// reduces the seven sums, and the last CTA to finish (ticket counter) writes the result.  Replaces four
// launches (gather, blur axis 0, blur axis 1 + sums, final) -- at BFGS problem sizes (1e4..1e6 events) the
// evaluation is launch-bound.
constexpr int kTileY = 8, kTileX = 32, kFusedMaxR = 8;

// Sharded evaluation (one process per GPU): every rank's partial planar images [3][Hc*Wc] (I, D0, D1) live in symmetric
// memory; the tail of EVERY rank reads all of them through NVLink peer pointers and sums them on the fly (in rank order, so all
// ranks compute bit-identical f and g) -- the all-reduce is fused into the objective kernel, there is no NCCL call.
constexpr int kMaxCmaxPeers = 16;
struct CmaxPeers {
    const float *img[kMaxCmaxPeers];                  // [3][Hc*Wc] per rank
    const unsigned long long *oob[kMaxCmaxPeers];     // out-of-canvas events per rank
    int world;
};

__device__ __forceinline__ float gather_peers(const CmaxPeers &P, int Hc, int Wc, int y, int x, int comp)
{
    const int64_t npix = (int64_t)Hc * Wc, i = (int64_t)comp * npix + (int64_t)y * Wc + x;
    float v = 0.f;
    for (int r = 0; r < P.world; ++r) v += __ldcg(P.img[r] + i);       // peer loads bypass L1 (the data was written by another GPU)
    return v;
}

__device__ __forceinline__ float gather_pixel(const float *acc, const float *planar, int replicas, int Hc, int Wc, int y, int x, int comp)
{
    // comp 0: I, 1: D0, 2: D1 (see cmax_gather_kernel for the block / sign conventions)
    const int64_t npix = (int64_t)Hc * Wc;
    float v = (comp == 0 && planar) ? planar[(int64_t)y * Wc + x] : 0.f;
    for (int r = 0; r < replicas; ++r) {
        const float *base = acc + (int64_t)r * npix * kBlockFloats;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int by = y - (k >> 1), bx = x - (k & 1);
            if (by < 0 || bx < 0) continue;
            const float *blk = base + ((int64_t)by * Wc + bx) * kBlockFloats;
            if (comp == 0) v += blk[k];
            else if (comp == 1) v += (k == 0) ? -blk[4] : (k == 1) ? blk[4] : (k == 2) ? -blk[5] : blk[5];
            else v += (k == 0) ? -blk[6] : (k == 1) ? -blk[7] : (k == 2) ? blk[6] : blk[7];
        }
    }
    return v;
}

template <bool PEER>
__global__ void __launch_bounds__(kTileY *kTileX) cmax_fused_var_tail_kernel_t(const CmaxPeers PE, const float *__restrict__ acc, const float *__restrict__ planar, int replicas, int Hc, int Wc,
                                                                              const BlurTaps taps, int do_blur, int want_grad,
                                                                              double mix_a, double mix_b, float *__restrict__ iwe_out,
                                                                              float *__restrict__ diwe_out, double *sums,
                                                                              unsigned *ticket, const unsigned long long *oob,
                                                                              double *result, double *partials = nullptr)
{
    __shared__ float tileI[(kTileY + 2 * kFusedMaxR) * (kTileX + 2 * kFusedMaxR)];
    __shared__ float tileT[kTileY * (kTileX + 2 * kFusedMaxR)];
    // blockIdx.z = candidate index of a batched evaluation: its own accumulator, sums, ticket and result
    acc += (size_t)blockIdx.z * (size_t)Hc * Wc * kBlockFloats * replicas;
    sums += 8 * blockIdx.z;
    ticket += blockIdx.z;
    result += 12 * blockIdx.z;
    const int r = do_blur ? taps.r : 0;
    const int hw = kTileX + 2 * r, hh = kTileY + 2 * r;
    const int y0 = blockIdx.y * kTileY, x0 = blockIdx.x * kTileX;
    const int tid = threadIdx.y * kTileX + threadIdx.x;
    // 1. halo tile of the un-blurred IWE
    for (int j = tid; j < hh * hw; j += kTileY * kTileX) {
        const int ly = j / hw, lx = j - ly * hw;
        const int gy = reflect_idx(y0 - r + ly, Hc), gx = reflect_idx(x0 - r + lx, Wc);
        tileI[j] = PEER ? gather_peers(PE, Hc, Wc, gy, gx, 0) : gather_pixel(acc, planar, replicas, Hc, Wc, gy, gx, 0);
    }
    const int y = y0 + threadIdx.y, x = x0 + threadIdx.x;
    const bool inside = y < Hc && x < Wc;
    float vi = 0.f, d0 = 0.f, d1 = 0.f;
    if (inside) {
        d0 = PEER ? gather_peers(PE, Hc, Wc, y, x, 1) : gather_pixel(acc, nullptr, replicas, Hc, Wc, y, x, 1);
        d1 = PEER ? gather_peers(PE, Hc, Wc, y, x, 2) : gather_pixel(acc, nullptr, replicas, Hc, Wc, y, x, 2);
    }
    __syncthreads();
    if (inside) {
        vi = tileI[(threadIdx.y + r) * hw + threadIdx.x + r];
        const int64_t npix = (int64_t)Hc * Wc, i = (int64_t)y * Wc + x;
        if (iwe_out) iwe_out[i] = vi;
        if (diwe_out) { diwe_out[i] = d0; diwe_out[npix + i] = d1; }
    }
    double g = (double)vi;
    if (do_blur) {
        // 2. axis 0 (vertical), every column of the halo; rounded to f32 like scipy's intermediate array
        for (int j = tid; j < kTileY * hw; j += kTileY * kTileX) {
            const int ly = j / hw, lx = j - ly * hw;
            const float *col = tileI + (ly + r) * hw + lx;
            double a = (double)col[0] * taps.w[0];
            for (int k = 1; k <= r; ++k) a += ((double)col[-k * hw] + (double)col[k * hw]) * taps.w[k];
            tileT[j] = (float)a;
        }
        __syncthreads();
        // 3. axis 1 (horizontal)
        const float *row = tileT + threadIdx.y * hw + threadIdx.x + r;
        double a = (double)row[0] * taps.w[0];
        for (int k = 1; k <= r; ++k) a += ((double)row[-k] + (double)row[k]) * taps.w[k];
        g = (double)(float)a;
    }
    if (!inside) { g = 0.0; vi = 0.f; }
    // 4. the seven sums (same slots as the separate kernels)
    const int cta = blockIdx.y * gridDim.x + blockIdx.x, nctas = gridDim.x * gridDim.y;
    if (PEER) {
        // sharded evaluation: every rank must arrive at bit-identical f and g (a BFGS driver runs replicated), so the sums
        // are formed in a fixed order: per-CTA partials to memory, the last CTA adds them up CTA by CTA
        const double v[7] = {(double)vi, g, g * g, g * (double)d0, g * (double)d1, (double)d0, (double)d1};
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const double sk = block_sum_ordered(v[k]);
            if (tid == 0) partials[(size_t)cta * 8 + k] = sk;
        }
    } else {
        block_add((double)vi, sums + 0);
        block_add(g, sums + 1);
        block_add(g * g, sums + 2);
        block_add(g * (double)d0, sums + 3);
        block_add(g * (double)d1, sums + 4);
        block_add((double)d0, sums + 5);
        block_add((double)d1, sums + 6);
    }
    // 5. last CTA writes the result
    __shared__ bool last;
    if (tid == 0) {
        __threadfence();
        last = atomicAdd(ticket, 1u) == (unsigned)nctas - 1;
    }
    __syncthreads();
    if (last && tid == 0) {
        __threadfence();
        double s[7];
        if (PEER) {
            for (int k = 0; k < 7; ++k) s[k] = 0.0;
            for (int c = 0; c < nctas; ++c)
                for (int k = 0; k < 7; ++k) s[k] += __ldcg(partials + (size_t)c * 8 + k);
        } else {
            for (int k = 0; k < 7; ++k) s[k] = atomicAdd(sums + k, 0.0);   // read through L2
        }
        const double P = (double)Hc * (double)Wc;
        const double mean_g = s[1] / P, var = s[2] / P - mean_g * mean_g, mu = s[0] / P;
        const double g0 = -2.0 * (s[3] - mu * s[5]) / P, g1 = -2.0 * (s[4] - mu * s[6]) / P;
        result[0] = -var;
        result[1] = want_grad ? (mix_a * g0 + mix_b * g1) : 0.0;
        result[2] = want_grad ? (mix_b * g0 + mix_a * g1) : 0.0;
        result[3] = s[0];
        if (PEER) {
            unsigned long long bad = 0;
            for (int r = 0; r < PE.world; ++r) bad += __ldcg(PE.oob[r]);
            result[4] = (double)bad;
        } else {
            result[4] = (double)(*oob);
        }
        result[5] = var;
        result[6] = g0;
        result[7] = g1;
    }
}

struct CmaxWorkspace {
    float *planar;              // on-chip path: planar IWE the CTAs' shared-memory images are bulk-reduced into
    float *acc, *I, *D0, *D1, *tmp, *G;
    double *bsums;              // [kMaxCandidates][8] sums of a batched evaluation
    unsigned *btickets;         // [kMaxCandidates]
    double *w, *wt;             // generic objectives: per-pixel weight image and its axis-0 blur
    double *gsums;              // 8 doubles (generic objectives)
    unsigned *gmax;             // order-preserving encoding of max(G)
    double *sums;               // 8 doubles
    unsigned long long *oob;    // 1
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static size_t carve(void *base, int Hs, int Ws, CmaxWorkspace *ws)
{
    const size_t npix = (size_t)(Hs + 1) * (Ws + 1);
    size_t off = 0;
    char *b = static_cast<char *>(base);
    auto take = [&](size_t bytes) { char *p = b ? b + off : nullptr; off += align_up(bytes, 256); return p; };
    // the small counters come first and are directly followed by the accumulator, so that ONE memset
    // zeroes counters + the R replicas an evaluation uses
    double *bsums = (double *)take(kMaxCandidates * 8 * sizeof(double));
    unsigned *btickets = (unsigned *)take(kMaxCandidates * sizeof(unsigned));
    double *gsums = (double *)take(8 * sizeof(double));
    unsigned *gmax = (unsigned *)take(sizeof(unsigned));
    double *sums = (double *)take(8 * sizeof(double));
    unsigned long long *oob = (unsigned long long *)take(sizeof(unsigned long long));
    float *planar = (float *)take(((npix + 3) & ~(size_t)3) * sizeof(float));
    float *acc = (float *)take(npix * kBlockFloats * sizeof(float) * (kMaxCandidates > kMaxReplicas ? kMaxCandidates : kMaxReplicas));
    float *I = (float *)take(npix * sizeof(float));
    float *D0 = (float *)take(npix * sizeof(float));
    float *D1 = (float *)take(npix * sizeof(float));
    float *tmp = (float *)take(npix * sizeof(float));
    float *G = (float *)take(npix * sizeof(float));
    double *w = (double *)take(npix * sizeof(double));
    double *wt = (double *)take(npix * sizeof(double));
    if (ws) {
        ws->planar = planar; ws->acc = acc; ws->I = I; ws->D0 = D0; ws->D1 = D1; ws->tmp = tmp; ws->G = G; ws->w = w; ws->wt = wt;
        ws->gsums = gsums; ws->gmax = gmax; ws->sums = sums; ws->oob = oob; ws->bsums = bsums; ws->btickets = btickets;
    }
    return off;
}

// channel-mix coefficients of scipy's blur along the length-2 stack axis (reflect):
// blurring the unit vector [1,0]: index i of the reflected signal equals 0 for i mod 4 in {0,3}.
static void mix_coeffs(const BlurTaps &t, double *a, double *b)
{
    double sa = 0.0, sb = 0.0;
    for (int k = -t.r; k <= t.r; ++k) {
        int i = k % 4;
        if (i < 0) i += 4;
        const double w = t.w[k < 0 ? -k : k];
        if (i == 0 || i == 3) sa += w; else sb += w;
    }
    *a = sa; *b = sb;
}

// The blur-sigma rule of every entry point that takes a sigma, applied before any CUDA call: NaN is an argument error,
// sigma <= 0 means no blur, and a positive sigma needs the truncate-4 radius (int)(4 sigma + 0.5) <= kMaxRadius.  The
// radius is compared in double, so no sigma (+inf, or one past the int range) can overflow the conversion.
static int check_sigma(const char *who, double sigma)
{
    if (sigma != sigma) { set_error("%s: blur sigma is NaN", who); return EVK_E_ARG; }
    const double r = 4.0 * sigma + 0.5;
    if (sigma > 0.0 && r >= (double)(kMaxRadius + 1)) {
        set_error("%s: blur sigma %.3f needs radius %.0f > %d", who, sigma, floor(r), kMaxRadius);
        return EVK_E_UNSUPPORTED;
    }
    return EVK_OK;
}

// taps of a blur with sigma > 0 (check_sigma's rule)
static int make_taps(double sigma, BlurTaps *t)
{
    int rc = check_sigma("evk_cmax", sigma);
    if (rc) return rc;
    const int r = (int)(4.0 * sigma + 0.5);
    t->r = r;
    double s = 0.0;
    for (int k = -r; k <= r; ++k) s += exp(-0.5 / (sigma * sigma) * (double)k * (double)k);
    for (int k = 0; k <= r; ++k) t->w[k] = exp(-0.5 / (sigma * sigma) * (double)k * (double)k) / s;
    return EVK_OK;
}

// image-space tail shared by the event entry points and the precomputed-image entry point
static int launch_tail(const CmaxWorkspace &ws, int Hc, int Wc, double sigma, unsigned flags, int objective, double obj_param,
                       bool grad, double *result, cudaStream_t st)
{
    const int npix = Hc * Wc;
    BlurTaps taps{};
    double mix_a = 1.0, mix_b = 0.0;
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
        if (!(flags & EVK_CMAX_NO_CHANNEL_MIX)) mix_coeffs(taps, &mix_a, &mix_b);
    }
    const int g = (npix + 255) / 256;
    if (do_blur) { prof_count(1); cmax_blur_axis0_kernel<<<g, 256, 0, st>>>(ws.I, ws.tmp, Hc, Wc, taps); }
    if (objective == OBJ_VARIANCE) {
        prof_count(2);
        cmax_blur_axis1_sums_kernel<<<g, 256, 0, st>>>(ws.tmp, ws.I, ws.D0, ws.D1, Hc, Wc, taps, do_blur, ws.sums);
        cmax_final_kernel<<<1, 1, 0, st>>>(ws.sums, ws.oob, npix, mix_a, mix_b, grad ? 1 : 0, result);
    } else {
        if (objective < OBJ_SOS || objective > OBJ_SOSA) { set_error("evk_cmax: unknown objective %d", objective); return EVK_E_ARG; }
        const bool g_needed = grad && objective != OBJ_MOA;
        prof_count(3);
        cmax_blur_axis1_store_kernel<<<g, 256, 0, st>>>(ws.tmp, ws.I, Hc, Wc, taps, do_blur, ws.G);
        cmax_obj_reduce_kernel<<<g, 256, 0, st>>>(ws.G, ws.I, npix, objective, obj_param, ws.gsums, ws.gmax, ws.w);
        if (g_needed) {
            prof_count(do_blur ? 2 : 1);
            if (do_blur) cmax_blur_d_axis0_kernel<<<g, 256, 0, st>>>(ws.w, ws.wt, Hc, Wc, taps);
            cmax_blur_d_axis1_dot_kernel<<<g, 256, 0, st>>>(ws.wt, ws.w, ws.D0, ws.D1, Hc, Wc, taps, do_blur, ws.gsums);
        }
        cmax_obj_final_kernel<<<1, 1, 0, st>>>(objective, ws.gsums, ws.gmax, ws.sums, ws.oob, npix, mix_a, mix_b, g_needed ? 1 : 0, result);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// event count from which the on-chip IWE pays for its fixed cost (174 KB of shared memory initialised and bulk-reduced per CTA;
// EVK_CMAX_ONCHIP_MIN overrides)
static int64_t onchip_min_events()
{
    static int64_t v = -1;
    if (v < 0) {
        const char *e = getenv("EVK_CMAX_ONCHIP_MIN");
        v = (e && *e) ? atoll(e) : ((int64_t)4 << 20);
    }
    return v;
}

// The event pass (pass 1): the on-chip fixed-point IWE from onchip_min_events() events up, the L2 block accumulator below
// that (EVK_VARIANT_SMEM_TILE / EVK_VARIANT_VECTOR_RED force one or the other).  Zeroes the counters, the planar image and
// the accumulator replicas it uses; leaves the replica count in A.replicas and the planar image (or null) in A.planar.
template <int WARP>
static int launch_event_pass(CmaxArgs &A, unsigned flags, bool grad, const CmaxWorkspace &ws, cudaStream_t st)
{
    const int Hs = A.Hc - 1, Ws = A.Wc - 1;
    const int npix = A.Hc * A.Wc;
    int R = (int)(A.n / (1 << 20));
    R = R < 1 ? 1 : (R > kMaxReplicas ? kMaxReplicas : R);
    A.replicas = R;
    A.acc = ws.acc;
    A.oob = ws.oob;
    // on-chip IWE: worth its fixed cost (174 KB of shared memory initialised and bulk-reduced per CTA) for
    // large event sets only; EVK_VARIANT_SMEM_TILE / EVK_VARIANT_VECTOR_RED force one or the other
    const size_t onchip_smem = (((size_t)npix + 3) & ~(size_t)3) * sizeof(float);
    const unsigned variant = variant_of(flags);
    bool onchip = onchip_smem <= (size_t)200 * 1024 && A.n > 0 &&
                  (variant == EVK_VARIANT_SMEM_TILE || (variant == EVK_VARIANT_AUTO && A.n >= onchip_min_events()));
    if (variant == EVK_VARIANT_VECTOR_RED || variant == EVK_VARIANT_GLOBAL_RED) onchip = false;
    A.planar = onchip ? ws.planar : nullptr;
    A.vec16 = ((((uintptr_t)A.x | (uintptr_t)A.y | (uintptr_t)A.t | (uintptr_t)A.p) & 15) == 0) ? 1 : 0;
    if (onchip && !grad) { R = 1; A.replicas = 1; }   // the blocks only receive carries and slow-path taps
    // counters (gsums, gmax, sums, oob), the planar image and the R accumulator replicas are contiguous: one memset
    EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)((char *)ws.acc - (char *)ws.gsums) + (size_t)R * npix * kBlockFloats * sizeof(float), st));
    if (WARP == WARP_FLOW_F32 && A.n > 0) {
        // the generic objectives' weight image (unused by the variance tail) holds the interleaved flow
        prof_count(1);
        launch_flow_interleave(A.flow, (int64_t)Hs * Ws, reinterpret_cast<float2 *>(ws.w), st);
        A.flow_uv = reinterpret_cast<const float2 *>(ws.w);
    }
    if (onchip) {
        ProfScope prof(st);
        prof_count(1);
        int64_t need_ctas = (A.n + kOnchipThreads * 8 - 1) / (kOnchipThreads * 8);
        const int g = (int)(need_ctas < num_sms() ? need_ctas : num_sms());
        if (grad) {
            EVK_CUDA(cudaFuncSetAttribute(cmax_onchip_kernel<WARP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)onchip_smem));
            cmax_onchip_kernel<WARP, true><<<g, kOnchipThreads, onchip_smem, st>>>(A);
        } else {
            EVK_CUDA(cudaFuncSetAttribute(cmax_onchip_kernel<WARP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)onchip_smem));
            cmax_onchip_kernel<WARP, false><<<g, kOnchipThreads, onchip_smem, st>>>(A);
        }
        EVK_CUDA(cudaGetLastError());
    } else if (A.n > 0) {
        ProfScope prof(st);
        prof_count(1);
        if (grad) cmax_scatter_kernel<WARP, true><<<grid_for(cmax_scatter_kernel<WARP, true>, 256, A.n, 256 * 4), 256, 0, st>>>(A);
        else cmax_scatter_kernel<WARP, false><<<grid_for(cmax_scatter_kernel<WARP, false>, 256, A.n, 256 * 4), 256, 0, st>>>(A);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// partial_images != nullptr: stop after the event pass and leave this rank's planar I, D0, D1 ([3][Hc*Wc]) and its
// out-of-canvas count there (the sharded evaluation's first half; evk_cmax_peer_tail_f32 is the second)
template <int WARP>
static int run_cmax(CmaxArgs A, double sigma, unsigned flags, int objective, double obj_param, double *result,
                    float *iwe_out, float *diwe_out, void *workspace, size_t workspace_bytes, cudaStream_t st,
                    float *partial_images = nullptr, unsigned long long *partial_oob = nullptr)
{
    const int Hs = A.Hc - 1, Ws = A.Wc - 1;
    if (A.n < 0 || Hs < 1 || Ws < 1 || (!result && !partial_images) || !workspace) { set_error("evk_cmax: bad arguments"); return EVK_E_ARG; }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_cmax: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hs, Ws, &ws);
    if (workspace_bytes < need) { set_error("evk_cmax: workspace of %zu bytes required, %zu given", need, workspace_bytes); return EVK_E_WORKSPACE; }
    const int npix = A.Hc * A.Wc;
    const bool grad = (flags & EVK_CMAX_WANT_GRAD) != 0 && WARP != WARP_FLOW_F32;
    A.abs_polarity = (flags & EVK_CMAX_ABS_POLARITY) ? 1 : 0;
    int rc = launch_event_pass<WARP>(A, flags, grad, ws, st);
    if (rc) return rc;
    const int R = A.replicas;
    const float *planar = A.planar;
    if (partial_images) {
        prof_count(1);
        cmax_gather_kernel<<<(npix + 255) / 256, 256, 0, st>>>(ws.acc, planar, R, A.Hc, A.Wc, partial_images, partial_images + npix,
                                                                partial_images + 2 * (size_t)npix, nullptr, nullptr, ws.sums, ws.oob, partial_oob);
        EVK_CUDA(cudaGetLastError());
        return EVK_OK;
    }
    BlurTaps taps{};
    double mix_a = 1.0, mix_b = 0.0;
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        rc = make_taps(sigma, &taps);
        if (rc) return rc;
        if (!(flags & EVK_CMAX_NO_CHANNEL_MIX)) mix_coeffs(taps, &mix_a, &mix_b);
    }
    if (objective == OBJ_VARIANCE && taps.r <= kFusedMaxR) {
        // launch-bound regime matters most here: gather + blur + sums + final in one kernel
        prof_count(1);
        dim3 tgrid((A.Wc + kTileX - 1) / kTileX, (A.Hc + kTileY - 1) / kTileY), tblock(kTileX, kTileY);
        cmax_fused_var_tail_kernel_t<false><<<tgrid, tblock, 0, st>>>(CmaxPeers{}, ws.acc, planar, R, A.Hc, A.Wc, taps, do_blur, grad ? 1 : 0, mix_a, mix_b, iwe_out,
                                                               diwe_out, ws.sums, ws.gmax, ws.oob, result);
        EVK_CUDA(cudaGetLastError());
        return EVK_OK;
    }
    prof_count(1);
    cmax_gather_kernel<<<(npix + 255) / 256, 256, 0, st>>>(ws.acc, planar, R, A.Hc, A.Wc, ws.I, ws.D0, ws.D1, iwe_out, diwe_out, ws.sums);
    return launch_tail(ws, A.Hc, A.Wc, sigma, flags, objective, obj_param, grad, result, st);
}

// Image-space tail of the motion models on the gathered IWE ws.I: blur, f and the side values into gsums / gmax, and
// (W_out != nullptr) the gradient pass's W = G(C) as f32 into W_out.
static int model_tail(const CmaxWorkspace &ws, int Hc, int Wc, double sigma, int objective, double obj_param, float *W_out,
                      cudaStream_t st)
{
    const int npix = Hc * Wc;
    BlurTaps taps{};
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
    }
    const int g = (npix + 255) / 256;
    prof_count(do_blur ? 3 : 2);
    if (do_blur) cmax_blur_axis0_kernel<<<g, 256, 0, st>>>(ws.I, ws.tmp, Hc, Wc, taps);
    cmax_blur_axis1_store_kernel<<<g, 256, 0, st>>>(ws.tmp, ws.I, Hc, Wc, taps, do_blur, ws.G);
    cmax_model_stats_kernel<<<g, 256, 0, st>>>(ws.G, ws.I, npix, objective, obj_param, ws.gsums, ws.gmax, W_out ? ws.w : nullptr, W_out);
    if (W_out && objective != OBJ_VARIANCE) {
        prof_count(do_blur ? 2 : 1);
        if (do_blur) cmax_blur_d_axis0_kernel<<<g, 256, 0, st>>>(ws.w, ws.wt, Hc, Wc, taps);
        cmax_blur_d_axis1_store_kernel<<<g, 256, 0, st>>>(ws.wt, ws.w, Hc, Wc, taps, do_blur, W_out);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// One evaluation of a motion model: pass 1 (IWE), the image-space tail, pass 2 (gradient) when asked for.
// The derivative planes D0 / D1 of the workspace are not used by this path: D0 holds W, sums[1..4] the gradient sums U.
template <int WARP>
static int run_model(CmaxArgs A, double sigma, unsigned flags, int objective, double obj_param, double *result, float *iwe_out,
                     void *workspace, size_t workspace_bytes, cudaStream_t st)
{
    const int Hs = A.Hc - 1, Ws = A.Wc - 1;
    if (A.n < 0 || Hs < 1 || Ws < 1 || !result || !workspace) { set_error("evk_cmax_warp: bad arguments"); return EVK_E_ARG; }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_cmax_warp: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    if (objective < OBJ_VARIANCE || objective > OBJ_SOSA) { set_error("evk_cmax_warp: unknown objective %d", objective); return EVK_E_ARG; }
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hs, Ws, &ws);
    if (workspace_bytes < need) { set_error("evk_cmax_warp: workspace of %zu bytes required, %zu given", need, workspace_bytes); return EVK_E_WORKSPACE; }
    const int npix = A.Hc * A.Wc;
    const size_t w_smem = (size_t)npix * sizeof(float);
    const bool grad = (flags & EVK_CMAX_WANT_GRAD) != 0 && objective != OBJ_MOA;
    if (grad && w_smem > (size_t)200 * 1024) {
        set_error("evk_cmax_warp: the gradient pass holds the %dx%d canvas in shared memory (at most 200 KB)", A.Hc, A.Wc);
        return EVK_E_UNSUPPORTED;
    }
    A.abs_polarity = (flags & EVK_CMAX_ABS_POLARITY) ? 1 : 0;
    int rc = launch_event_pass<WARP>(A, flags, false, ws, st);
    if (rc) return rc;
    prof_count(1);
    cmax_gather_kernel<<<(npix + 255) / 256, 256, 0, st>>>(ws.acc, A.planar, A.replicas, A.Hc, A.Wc, ws.I, ws.D0, ws.D1, iwe_out, nullptr, ws.sums);
    rc = model_tail(ws, A.Hc, A.Wc, sigma, objective, obj_param, grad ? ws.D0 : nullptr, st);
    if (rc) return rc;
    double *U = ws.sums + 1;
    if (grad && A.n > 0) {
        ProfScope prof(st);
        prof_count(1);
        int64_t need_ctas = (A.n + kGradThreads * 8 - 1) / (kGradThreads * 8);
        const int g = (int)(need_ctas < num_sms() ? need_ctas : num_sms());
        EVK_CUDA(cudaFuncSetAttribute(cmax_grad_pass_kernel<WARP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)w_smem));
        cmax_grad_pass_kernel<WARP><<<g, kGradThreads, w_smem, st>>>(A, ws.D0, U);
        EVK_CUDA(cudaGetLastError());
    }
    cmax_model_final_kernel<<<1, 1, 0, st>>>(objective, ws.gsums, ws.gmax, ws.sums, ws.oob, npix, U, model_dims(WARP), grad ? 1 : 0, result);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// host model array -> WarpModel (rotation: 3 doubles, xyztheta: 6)
static int read_model(int warp, const double *model, WarpModel *M, int *n_doubles)
{
    if (!model) { set_error("evk_cmax_warp: null model"); return EVK_E_ARG; }
    int nd;
    if (warp == EVK_WARP_ROTATION) nd = 3;
    else if (warp == EVK_WARP_XYZTHETA) nd = 6;
    else { set_error("evk_cmax_warp: unknown warp %d", warp); return EVK_E_ARG; }
    *M = WarpModel{};
    for (int k = 0; k < nd; ++k) M->m[k] = model[k];
    if (n_doubles) *n_doubles = nd;
    return EVK_OK;
}

// precomputed planar iwe / diwe -> the planar working images + their sums (the block accumulator is
// bypassed: a block value stands for taps of TWO pixels, planar images cannot be packed into it)
__global__ void __launch_bounds__(256) cmax_planar_kernel(const float *__restrict__ iwe, const float *__restrict__ diwe,
                                                          int npix, float *__restrict__ I, float *__restrict__ D0,
                                                          float *__restrict__ D1, double *sums)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    float a = 0.f, b = 0.f, c = 0.f;
    if (i < npix) {
        a = iwe[i];
        if (diwe) { b = diwe[i]; c = diwe[npix + i]; }
        I[i] = a; D0[i] = b; D1[i] = c;
    }
    block_add((double)a, sums + 0);
    block_add((double)b, sums + 5);
    block_add((double)c, sums + 6);
}

// ---- dense-flow objective over a batch of samples (evk_cmax_flow_objective_f32 / _grad_f32) -------------------------
// Sample b = events [offsets[b], offsets[b+1]) (clipped to [0, n)) warped by flow[b] (optic_flow.py:37-44), the bilinear
// IWE of draw_flow.py:18-21 on the (H+1)x(W+1) canvas keeping only events with 0 <= x' < W and 0 <= y' < H, the blur and
// one of the objectives of objectives.py:231-236, 308-400, 478-523.  The grid of both event passes is (slices, batch):
// blockIdx.y is the sample, so no event searches for its sample and the launch count does not depend on the batch.
//   forward:  one v4 reduction per kept event into the sample's 2x2-block image [B][Hc][Wc][4] (16 B per pixel)
//   backward: W = g_b G(C_b) per sample (C = df/dG), then per event the four taps of W (L2 gathers) give df/dx', df/dy';
//             times d they are spread over the event's four grid_sample taps: two v4 reductions into the 2x2-block
//             flow gradient [B][2][H][W][4] of evk_warp_flow_grad_f32.
//
// ---- what every batched event pass shares (dense flow, parametric motion, segmentation, timestamp losses) ----------
// The event arrays the batched passes read.  Sample b is events [offsets[b], offsets[b+1]), clipped to [0, n).
struct EventSource {
    const float *x, *y, *t, *p;  // t relative to the sample's t0
    const float *tau;            // the timestamp losses: the normalised stamp of every event
    const int64_t *offsets;
    int64_t n;
    const float *rho;            // the camera motion: the inverse depth of every event (null for the other models)
};

__device__ __forceinline__ void sample_range(const EventSource &E, int b, int64_t &first, int64_t &last)
{
    first = E.offsets[b];
    last = E.offsets[b + 1];
    if (first < 0) first = 0;
    if (last > E.n) last = E.n;
}

// The record of one event that a pass reads, and its loaders
struct EvXYT { float x, y, t; };
struct EvXYTP { float x, y, t, p; };
struct EvXYTUP { float x, y, t, tau, p; };
struct EvXYTPW { float x, y, t, p, w; };

__device__ __forceinline__ EvXYT load_xyt(const EventSource &E, int64_t i)
{
    return {ld_stream(E.x + i), ld_stream(E.y + i), ld_stream(E.t + i)};
}
__device__ __forceinline__ EvXYTP load_xytp(const EventSource &E, int64_t i)
{
    return {ld_stream(E.x + i), ld_stream(E.y + i), ld_stream(E.t + i), ld_stream(E.p + i)};
}
__device__ __forceinline__ EvXYTUP load_xytup(const EventSource &E, int64_t i)
{
    return {ld_stream(E.x + i), ld_stream(E.y + i), ld_stream(E.t + i), ld_stream(E.tau + i), ld_stream(E.p + i)};
}

// A record of the loaders above with, for a model whose events carry it (has_depth), the event's inverse depth: the
// other models' records stay what they were.  depth_of reads it back (0 without).
template <class Rec, bool DEPTH>
struct Depthed : Rec {};
template <class Rec>
struct Depthed<Rec, true> : Rec {
    float rho;
};

template <int WARP, class Rec>
__device__ __forceinline__ Depthed<Rec, has_depth(WARP)> with_depth(const EventSource &E, int64_t i, const Rec &r)
{
    Depthed<Rec, has_depth(WARP)> q;
    static_cast<Rec &>(q) = r;
    if constexpr (has_depth(WARP)) q.rho = ld_stream(E.rho + i);
    return q;
}
template <class Rec>
__device__ __forceinline__ float depth_of(const Depthed<Rec, false> &) { return 0.0f; }
template <class Rec>
__device__ __forceinline__ float depth_of(const Depthed<Rec, true> &r) { return r.rho; }

constexpr int kFlowObjThreads = 256;

// The event loop of a single-model pass over [first, last) on the (slices, batch) grid: kBatch records loaded per thread
// before any is used (see kBatch), then body(i, record) for each; the tail one event at a time.
template <class Load, class Body>
__device__ __forceinline__ void for_each_event(int64_t first, int64_t last, Load load, Body body)
{
    const int64_t stride = (int64_t)gridDim.x * kFlowObjThreads;
    int64_t i = first + (int64_t)blockIdx.x * kFlowObjThreads + threadIdx.x;
    for (; i + (kBatch - 1) * stride < last; i += kBatch * stride) {
        decltype(load(i)) e[kBatch];
#pragma unroll
        for (int k = 0; k < kBatch; ++k) e[k] = load(i + k * stride);
#pragma unroll
        for (int k = 0; k < kBatch; ++k) body(i + k * stride, e[k]);
    }
    for (; i < last; i += stride) body(i, load(i));
}

// The event loop of a multi-model pass: every batch is kBatch masked loads (the records past `last` keep their default
// value), then body(records, ne) with the ne records loaded, which runs every model over them.
template <class Load, class Body>
__device__ __forceinline__ void for_each_event_batch(int64_t first, int64_t last, Load load, Body body)
{
    const int64_t stride = (int64_t)gridDim.x * kFlowObjThreads;
    for (int64_t i = first + (int64_t)blockIdx.x * kFlowObjThreads + threadIdx.x; i < last; i += kBatch * stride) {
        decltype(load(i)) e[kBatch];
        int ne = 0;
#pragma unroll
        for (int k = 0; k < kBatch; ++k) {
            const int64_t q = i + k * stride;
            if (q < last) {
                e[k] = load(q);
                ne = k + 1;
            }
        }
        body(e, ne);
    }
}

// Model `index` of params [..][K] into M as model_taps reads it (xyztheta, the planar models and the camera rotation
// also take the fixed centre, behind their K parameters), and `count` consecutive models from `first` into shared
// memory for the whole CTA.  M is filled in place: a model returned by value costs the linvel forward pass two registers.
template <int WARP>
__device__ __forceinline__ void load_model(const double *params, int64_t index, double cx, double cy, ModelOf<WARP> &M)
{
    constexpr int K = model_dims(WARP);
    M = ModelOf<WARP>{};
#pragma unroll
    for (int k = 0; k < K; ++k) M.m[k] = params[index * K + k];
    if (!is_linvel(WARP) && !is_rotation(WARP)) { M.m[K] = cx; M.m[K + 1] = cy; }
}

template <int WARP>
__device__ __forceinline__ void load_models(const double *params, int64_t first, int count, double cx, double cy,
                                            ModelOf<WARP> *mod)
{
    for (int q = threadIdx.x; q < count; q += kFlowObjThreads) {
        ModelOf<WARP> M;
        load_model<WARP>(params, first + q, cx, cy, M);
        mod[q] = M;
    }
    __syncthreads();
}

// an event of the (f32) model passes, splatted with weight p; rho is its inverse depth, which only the camera motion's
// events carry
template <int WARP>
__device__ __forceinline__ Event<WARP> model_event(float x, float y, float t, float p, float rho = 0.0f)
{
    Event<WARP> e;
    e.x = x; e.y = y; e.t = t; e.p = p;
    if constexpr (has_depth(WARP)) e.rho = rho;
    return e;
}

// The accumulator of the timestamp losses.  Polarity image s of an event: 0 for p > 0, 1 for p <= 0, -1 for a NaN p,
// which is in neither image (evk_tsimg.cu).
__device__ __forceinline__ int ts_polarity(float p) { return p > 0.0f ? 0 : p <= 0.0f ? 1 : -1; }

// One event's taps into the sample's [2][Hc][Wc][8]: the 32-byte block {S taps, C taps} at the footprint's anchor in image
// s, tsimg_scatter_kernel's taps tau (1-dx)(1-dy) .. and (1-dx)(1-dy) ..
__device__ __forceinline__ void ts_block_add(float *acc, int64_t npix, int Wc, int s, const Taps &T, float tau)
{
    const float dx = T.dx, dy = T.dy;
    const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
    const float tl = __fmul_rn(tau, ox), tr = __fmul_rn(tau, dx);
    float *blk = acc + ((s ? npix : 0) + (int64_t)T.y0 * Wc + T.x0) * 8;
    red_add4(blk, make_float4(__fmul_rn(tl, oy), __fmul_rn(tr, oy), __fmul_rn(tl, dy), __fmul_rn(tr, dy)));
    red_add4(blk + 4, make_float4(__fmul_rn(ox, oy), __fmul_rn(dx, oy), __fmul_rn(ox, dy), __fmul_rn(dx, dy)));
}

// 16-byte accumulator blocks per image of the timestamp losses: one 32-byte block per canvas pixel and polarity; the
// dense-flow backward's flow-gradient blocks ([2][H][W] per sample) are fewer
static size_t flow_ts_acc_blocks(int H, int W) { return (size_t)2 * (H + 1) * (W + 1); }

// ---- the dense-flow passes ----
struct FlowArgs {
    CmaxArgs C;            // canvas (Hc, Wc) for splat_taps
    EventSource E;
    const float *flow;     // [B][2][H][W]
    int H, W;
    float *acc;            // forward: the sample's blocks ([B][Hc][Wc][4] or [B][2][Hc][Wc][8]); backward: [B][2][H][W][4]
    unsigned *nonfinite;   // [B] forward: set when an event's warped position is not finite
    const float *Wimg;     // contrast backward: [B][Hc][Wc]
    const float2 *ab;      // timestamp backward: (A, B) [B][2][Hc][Wc]
};

// The warp by the flow (u, v) at the event, the keep rule and the taps of one event; false for events that contribute
// nothing.  Shared by the dense-flow and the grid-flow passes.
__device__ __forceinline__ bool flow_obj_keep(const FlowArgs &A, float xe, float ye, float u, float v, float d, float p, Taps &T,
                                              bool &nonfinite)
{
    const float xw = __fadd_rn(xe, __fmul_rn(u, d)), yw = __fadd_rn(ye, __fmul_rn(v, d));
    if (!isfinite(xw) || !isfinite(yw)) { nonfinite = true; return false; }
    if (!(xw >= 0.0f && xw < (float)A.W && yw >= 0.0f && yw < (float)A.H)) return false;
    unsigned oob = 0;   // a kept event's footprint lies inside the canvas
    return splat_taps<false>(A.C, xw, yw, p, 0.0f, true, oob, T);
}

// The warp and the keep rule of one event of sample b; false for events that contribute nothing.
__device__ __forceinline__ bool flow_obj_warp(const FlowArgs &A, const float *flow, float xe, float ye, float d, float p,
                                              FlowSample &s, Taps &T, bool &nonfinite)
{
    s = flow_sample<false>(flow, nullptr, A.H, A.W, xe, ye);
    return flow_obj_keep(A, xe, ye, s.u, s.v, d, p, T, nonfinite);
}

// The backward of the flow losses: an event's df/dflow = (gu, gv) times the weights of its four grid_sample taps, added to
// the 2x2-block flow gradient acc [2][H][W][4] of its sample; taps outside the field get nothing.
__device__ __forceinline__ void flow_obj_spread(const FlowArgs &A, float *acc, const FlowSample &s, float gu, float gv)
{
    if (!s.sampled || (gu == 0.0f && gv == 0.0f)) return;
    const int64_t plane4 = (int64_t)A.H * A.W * 4;
    if (s.x0 >= 0 && s.x0 + 1 < A.W && s.y0 >= 0 && s.y0 + 1 < A.H) {
        float *blk = acc + ((int64_t)s.y0 * A.W + s.x0) * 4;
        red_add4(blk, make_float4(gu * s.nw, gu * s.ne, gu * s.sw, gu * s.se));
        red_add4(blk + plane4, make_float4(gv * s.nw, gv * s.ne, gv * s.sw, gv * s.se));
    } else {
        // border footprint: every tap inside the field is the TL tap of its own pixel's block
        const int xs[4] = {s.x0, s.x0 + 1, s.x0, s.x0 + 1}, ys[4] = {s.y0, s.y0, s.y0 + 1, s.y0 + 1};
        const float w[4] = {s.nw, s.ne, s.sw, s.se};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if ((unsigned)xs[k] >= (unsigned)A.W || (unsigned)ys[k] >= (unsigned)A.H) continue;
            float *blk = acc + ((int64_t)ys[k] * A.W + xs[k]) * 4;
            red_add(blk, gu * w[k]);
            red_add(blk + plane4, gv * w[k]);
        }
    }
}

template <bool GRAD>
__device__ __forceinline__ void flow_obj_event(const FlowArgs &A, const float *flow, float *acc, const float *Wb, const EvXYTP &e,
                                               bool &nonfinite)
{
    FlowSample s;
    Taps T;
    if (!flow_obj_warp(A, flow, e.x, e.y, e.t, e.p, s, T, nonfinite)) return;
    if (!GRAD) {
        red_add4(acc + ((int64_t)T.y0 * A.C.Wc + T.x0) * 4, T.ti);
        return;
    }
    // df/dx' and df/dy' through the four bilinear taps of the IWE (the sx / sy of cmax_grad_pass_kernel)
    const int r0 = T.y0 * A.C.Wc, r1 = T.y1 * A.C.Wc;
    const float w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0), w11 = __ldg(Wb + r1 + T.x1);
    const float ox = 1.0f - T.dx, oy = 1.0f - T.dy;
    float sx, sy;
    tap_slopes(ox, oy, T.dx, T.dy, w00, w01, w10, w11, sx, sy);
    flow_obj_spread(A, acc, s, T.wm * sx * e.t, T.wm * sy * e.t);
}

template <bool GRAD>
__global__ void __launch_bounds__(kFlowObjThreads) flow_obj_event_kernel(const FlowArgs A)
{
    const int b = blockIdx.y;
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int64_t npix = (int64_t)A.C.Hc * A.C.Wc;
    const float *flow = A.flow + (int64_t)b * 2 * A.H * A.W;
    float *acc = A.acc + (GRAD ? (int64_t)b * 2 * A.H * A.W * 4 : (int64_t)b * npix * 4);
    const float *Wb = GRAD ? A.Wimg + (int64_t)b * npix : nullptr;
    bool nonfinite = false;
    for_each_event(first, last, [&](int64_t i) { return load_xytp(A.E, i); },
                   [&](int64_t, const EvXYTP &e) { flow_obj_event<GRAD>(A, flow, acc, Wb, e, nonfinite); });
    if (!GRAD && nonfinite) A.nonfinite[b] = 1u;
}

// blocks -> the IWE of every sample (blockIdx.z); a sample with a non-finite warped position gets an all-NaN IWE, so that
// its f (and its gradient) is NaN
__global__ void __launch_bounds__(256) flow_obj_fold_kernel(const float *__restrict__ acc, const unsigned *__restrict__ nonfinite,
                                                            int Hc, int Wc, float *__restrict__ iwe)
{
    const int64_t npix = (int64_t)Hc * Wc;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    acc += blockIdx.z * npix * 4;
    const int y = i / Wc, x = i - y * Wc;
    float v = acc[(int64_t)i * 4];
    if (x > 0) v += acc[(int64_t)(i - 1) * 4 + 1];
    if (y > 0) v += acc[(int64_t)(i - Wc) * 4 + 2];
    if (x > 0 && y > 0) v += acc[(int64_t)(i - Wc - 1) * 4 + 3];
    iwe[blockIdx.z * npix + i] = nonfinite[blockIdx.z] ? __int_as_float(0x7fc00000) : v;
}

// f of every sample from the sums of cmax_model_stats_kernel (gsums[b][8]: 1 sum(exp G), 2 sum(exp(-p G)), 4 sum(G),
// 5 sum(G^2) with f64 products)
__global__ void flow_obj_final_kernel(int kind, const double *gsums, int npix, int batch, double *f_out)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    const double *s = gsums + 8 * b;
    const double P = (double)npix;
    double f;
    if (kind == OBJ_VARIANCE) { const double m = s[4] / P; f = -(s[5] / P - m * m); }
    else if (kind == OBJ_SOS) f = -s[5] / P;
    else if (kind == OBJ_SOE) f = -s[1] / P;
    else f = -s[2];
    f_out[b] = f;
}

// g_b * df_b/dG per pixel (before the blur that turns it into W):
//   variance -2 G / P (the -2 mean(G) / P of the exact derivative is constant over the image; the blur keeps it constant
//   and the tap differences of the event pass cancel it), sos -2 G / P, soe -exp(G) / P, sosa p exp(-p G)
__global__ void __launch_bounds__(256) flow_obj_coef_kernel(const float *__restrict__ G, int npix, int kind, double param,
                                                            const float *__restrict__ grad_f, double *__restrict__ w)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    const size_t k = (size_t)blockIdx.z * npix + i;
    const double g = (double)G[k], P = (double)npix;
    double c;
    if (kind == OBJ_SOE) c = -exp(g) / P;
    else if (kind == OBJ_SOSA) c = param * exp(-param * g);
    else c = -2.0 * g / P;
    w[k] = (double)grad_f[blockIdx.z] * c;
}

// [B][2][H][W][4] blocks -> grad_flow [B][2][H][W]
__global__ void __launch_bounds__(256) flow_obj_grad_fold_kernel(const float *__restrict__ ws, float *__restrict__ out, int64_t planes,
                                                                 int H, int W)
{
    const int64_t total = planes * H * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        float v = ws[i * 4];
        if (x > 0) v += ws[(i - 1) * 4 + 1];
        if (y > 0) v += ws[(i - W) * 4 + 2];
        if (x > 0 && y > 0) v += ws[(i - W - 1) * 4 + 3];
        out[i] = v;
    }
}

// ---- shared by the batched objectives (dense flow above, parametric motion below): workspace, checks, image tail ----
struct BatchObjWorkspace {
    unsigned *nonfinite;   // [B]
    double *gsums;         // [B][8]
    unsigned *gmax;        // [B]
    float *acc;            // [B][acc_blocks][4]: the 2x2-block IWE (forward); the flow objective's flow-gradient blocks
    float *tmp, *G, *Wimg; // [B][Hc][Wc]
    double *w, *wt;        // [B][Hc][Wc]
};

// acc_blocks: 16-byte blocks of the accumulator per sample.  Without `backward` the two f64 images of the adjoint blur
// are not carved (a forward-only entry, which may use Wimg for its folded images).
static size_t batch_obj_carve(void *base, int batch, int H, int W, size_t acc_blocks, BatchObjWorkspace *ws, bool backward = true)
{
    const size_t npix = (size_t)(H + 1) * (W + 1), B = (size_t)batch;
    size_t off = 0;
    char *b = static_cast<char *>(base);
    auto take = [&](size_t bytes) { char *p = b ? b + off : nullptr; off += align_up(bytes, 256); return p; };
    // the counters come first and are directly followed by the accumulator: one memset zeroes them all
    unsigned *nonfinite = (unsigned *)take(B * sizeof(unsigned));
    double *gsums = (double *)take(B * 8 * sizeof(double));
    unsigned *gmax = (unsigned *)take(B * sizeof(unsigned));
    float *acc = (float *)take(B * acc_blocks * 4 * sizeof(float));
    float *tmp = (float *)take(B * npix * sizeof(float));
    float *G = (float *)take(B * npix * sizeof(float));
    float *Wimg = (float *)take(B * npix * sizeof(float));
    double *w = backward ? (double *)take(B * npix * sizeof(double)) : nullptr;
    double *wt = backward ? (double *)take(B * npix * sizeof(double)) : nullptr;
    if (ws) { ws->nonfinite = nonfinite; ws->gsums = gsums; ws->gmax = gmax; ws->acc = acc; ws->tmp = tmp; ws->G = G; ws->Wimg = Wimg; ws->w = w; ws->wt = wt; }
    return off;
}

// The canvas every batched objective needs: H, W >= 2 and at most 2^30 canvas pixels (H+1)(W+1), so that pixel counts and
// indices fit an int.
static bool batch_canvas_ok(int H, int W)
{
    return H >= 2 && W >= 2 && (int64_t)(H + 1) * (W + 1) <= (int64_t)1 << 30;
}

// The limits of the dense-flow and model entries, which their workspace queries share.  `images` tail images per canvas
// (1 for the contrast losses, 2 for the timestamp losses), and at most 65535 images: 0 <= batch <= 65535 / images.
// n_cand 0: one canvas per sample; else n_cand forward-only canvases per sample, 1 <= n_cand <= kMaxCandidates and
// batch n_cand <= 65535 / images.
static bool batch_limits(int batch, int n_cand, int H, int W, int images)
{
    const int64_t max_batch = 65535 / images;
    if (batch < 0 || batch > max_batch || !batch_canvas_ok(H, W)) return false;
    return !n_cand || (n_cand >= 1 && n_cand <= kMaxCandidates && (int64_t)batch * n_cand <= max_batch);
}

// the flow objective's accumulator: the IWE blocks (forward) or the flow-gradient blocks (backward), whichever is larger
static size_t flow_obj_acc_blocks(int H, int W)
{
    const size_t npix = (size_t)(H + 1) * (W + 1), grad = (size_t)2 * H * W;
    return npix > grad ? npix : grad;
}

// the checks and set-up every batched objective entry shares: objective, canvas, workspace (carved into ws), blur taps
static int batch_obj_check(const char *who, const char *wrt, int batch, int H, int W, double sigma, int objective, size_t acc_blocks,
                           void *workspace, size_t workspace_bytes, BatchObjWorkspace &ws, BlurTaps &taps, bool backward = true)
{
    if (objective == OBJ_MOA || objective == OBJ_ISOA) {
        set_error("%s: objective %d (moa / isoa) is piecewise constant in the %s and has no gradient", who, objective, wrt);
        return EVK_E_UNSUPPORTED;
    }
    if (objective != OBJ_VARIANCE && objective != OBJ_SOS && objective != OBJ_SOE && objective != OBJ_SOSA) {
        set_error("%s: unknown objective %d", who, objective);
        return EVK_E_ARG;
    }
    const size_t need = batch_obj_carve(nullptr, batch, H, W, acc_blocks, nullptr, backward);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 255)) {
        set_error("%s: 256-byte aligned workspace of %zu bytes required", who, need);
        return EVK_E_WORKSPACE;
    }
    batch_obj_carve(workspace, batch, H, W, acc_blocks, &ws, backward);
    taps = BlurTaps{};
    if (sigma > 0.0) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
    }
    return EVK_OK;
}

// Shared argument checks and set-up of the dense-flow entries.  `images` per sample: 1 for the contrast losses, 2 for the
// timestamp losses (one per polarity; they also need tau), so that the tail's 65535 images allow 65535 or 32767 samples.
// acc_blocks: 16-byte accumulator blocks per image (batch_obj_carve).
static int flow_setup(const char *who, const float *x, const float *y, const float *t, const float *tau, const float *p,
                      const int64_t *offsets, int batch, int64_t n, const float *flow, int H, int W, double sigma, int objective,
                      int images, size_t acc_blocks, void *workspace, size_t workspace_bytes, FlowArgs &A, BatchObjWorkspace &ws,
                      BlurTaps &taps)
{
    if (int rc = check_sigma(who, sigma)) return rc;
    const int max_batch = 65535 / images;
    if (!batch_limits(batch, 0, H, W, images) || n < 0 || (batch > 0 && (!offsets || !flow)) ||
        (n > 0 && (!x || !y || !t || (images == 2 && !tau) || !p))) {
        set_error("%s: bad arguments (0 <= batch <= %d, H, W >= 2, (H+1)(W+1) <= 2^30)", who, max_batch);
        return EVK_E_ARG;
    }
    int rc = batch_obj_check(who, "flow", images * batch, H, W, sigma, objective, acc_blocks, workspace, workspace_bytes, ws, taps);
    if (rc) return rc;
    A = FlowArgs{};
    A.C.Hc = H + 1; A.C.Wc = W + 1;
    A.E = EventSource{x, y, t, p, tau, offsets, n};
    A.flow = flow; A.H = H; A.W = W;
    A.acc = ws.acc;
    A.nonfinite = ws.nonfinite;
    return EVK_OK;
}

// Zero the counters and the accumulators of `canvases` canvases of npix pixels, `floats` floats per pixel, before a forward
// event pass (batch_obj_carve puts them back to back)
static cudaError_t batch_obj_zero(const BatchObjWorkspace &ws, int64_t canvases, int npix, int floats, cudaStream_t st)
{
    return cudaMemsetAsync(ws.nonfinite, 0, (size_t)((char *)ws.acc - (char *)ws.nonfinite) + (size_t)canvases * npix * floats * sizeof(float),
                           st);
}

// (slices, batch) grid of every batched event pass: about 2K events per CTA, at most ~8 CTAs per SM over the whole batch
static dim3 batch_grid(int64_t n, int batch)
{
    const int64_t per = n / batch;
    int64_t slices = (per + 2047) / 2048;
    const int64_t fill = ((int64_t)num_sms() * 8 + batch - 1) / batch;
    if (slices > fill) slices = fill;
    if (slices < 1) slices = 1;
    return dim3((unsigned)slices, (unsigned)batch);
}

// G = blur(I) for every sample (blockIdx.z), both axes
static void batch_obj_blur(const BatchObjWorkspace &ws, const float *I, int Hc, int Wc, const BlurTaps &taps, int batch, cudaStream_t st)
{
    const int do_blur = taps.r > 0 || taps.w[0] != 0.0;
    const dim3 g((Hc * Wc + 255) / 256, 1, batch);
    prof_count(do_blur ? 2 : 1);
    if (do_blur) cmax_blur_axis0_kernel<<<g, 256, 0, st>>>(I, ws.tmp, Hc, Wc, taps);
    cmax_blur_axis1_store_kernel<<<g, 256, 0, st>>>(ws.tmp, I, Hc, Wc, taps, do_blur, ws.G);
}

// forward tail after the event pass: the 2x2-block images in ws.acc -> iwe_out (NaN for a sample flagged in ws.nonfinite),
// its blur and f of every sample
static void batch_obj_forward_tail(const BatchObjWorkspace &ws, int Hc, int Wc, const BlurTaps &taps, int batch, int objective,
                                   double obj_param, float *iwe_out, double *f_out, cudaStream_t st)
{
    const int npix = Hc * Wc;
    const dim3 g((npix + 255) / 256, 1, batch);
    prof_count(1);
    flow_obj_fold_kernel<<<g, 256, 0, st>>>(ws.acc, ws.nonfinite, Hc, Wc, iwe_out);
    batch_obj_blur(ws, iwe_out, Hc, Wc, taps, batch, st);
    prof_count(2);
    cmax_model_stats_kernel<<<g, 256, 0, st>>>(ws.G, iwe_out, npix, objective, obj_param, ws.gsums, ws.gmax, nullptr, nullptr);
    flow_obj_final_kernel<<<(batch + 127) / 128, 128, 0, st>>>(objective, ws.gsums, npix, batch, f_out);
}

// first half of a backward: W_b = G(grad_f[b] df_b/dG) into ws.Wimg, with G recomputed from the saved IWE
static void batch_obj_backward_W(const BatchObjWorkspace &ws, const float *iwe, int Hc, int Wc, const BlurTaps &taps, int batch,
                                 int objective, double obj_param, const float *grad_f, cudaStream_t st)
{
    const int npix = Hc * Wc;
    batch_obj_blur(ws, iwe, Hc, Wc, taps, batch, st);
    const int do_blur = taps.r > 0 || taps.w[0] != 0.0;
    const dim3 g((npix + 255) / 256, 1, batch);
    prof_count(do_blur ? 3 : 2);
    flow_obj_coef_kernel<<<g, 256, 0, st>>>(ws.G, npix, objective, obj_param, grad_f, ws.w);
    if (do_blur) cmax_blur_d_axis0_kernel<<<g, 256, 0, st>>>(ws.w, ws.wt, Hc, Wc, taps);
    cmax_blur_d_axis1_store_kernel<<<g, 256, 0, st>>>(ws.wt, ws.w, Hc, Wc, taps, do_blur, ws.Wimg);
}

// ---- grid-parametrised flow objective over a batch of samples (evk_cmax_grid_flow_*) --------------------------------
// The dense-flow objective with the flow of sample b given on a gh x gw grid of nodes (align_corners: node (i, j) at pixel
// (j (W-1)/(gw-1), i (H-1)/(gh-1))): an event at (x, y) takes the bilinear interpolation of the nodes at
// (x (gw-1)/(W-1), y (gh-1)/(H-1)), zero outside the node grid; then flow_obj_keep, the splat and the tail of the flow
// objective (optic_flow.py:37-44, draw_flow.py:15-26).  The grid of the event passes is (slices, batch), as for the
// flow objective, and every CTA holds its sample's nodes in dynamic shared memory as {u, v} pairs:
//   forward / candidates: grid_flow_cand_kernel.  Per event one 16-byte record, the node cell and its four weights once
//             (they do not depend on the candidate), then per candidate j four 8-byte node gathers from shared memory,
//             the warp and one v4 reduction into canvas z = b J + j, scored by batch_obj_forward_tail.
//   backward: batch_obj_backward_W, then grid_flow_grad_kernel: per event the four gathers of W_b give df/dx', df/dy'
//             (as in flow_obj_event); times t_rel and the four node weights they go to a per-CTA f64 accumulator
//             [2][gh][gw] in shared memory.  Coarse grids send a whole warp to a few node cells, and shared f32 / f64
//             adds are CAS loops on sm_90a, so the lanes of a warp with the same cell first sum their eight values
//             (match.any, then a shuffle tree over the peers) and one lane per cell adds them.  At the end one f64
//             atomic per node component and CTA into [B][2][gh][gw] (in the workspace), then a cast to the f32 output:
//             no L2 reduction per event and no per-pixel gradient blocks.
// The grid-flow average-timestamp loss (evk_grid_flow_timestamp_*) runs the same passes with TS = true: a 20-byte record
// per event, weight 1, the two v4 reductions of ts_block_add into image pair z = 2 (b J + j) + s and ts_obj_forward_tail;
// its backward gathers the (A, B) pairs of ts_obj_backward_ab instead of W_b, as flow_ts_event does.
constexpr int kMaxGridNodes = 4096;       // gh gw of the forward and backward
constexpr int kMaxGridCandNodes = 12288;   // n_cand gh gw of the candidates pass (96 KB of f32 nodes)

struct GridArgs {
    FlowArgs F;            // canvas, events, H, W, acc, nonfinite, Wimg
    const float *grid;     // [B][J][2][gh][gw]
    int gh, gw, J;
    float rx, ry;          // (gw-1)/(W-1), (gh-1)/(H-1) in f32
    double *grad;          // backward: [B][2][gh][gw]
};

// The node cell of an event: the shared-memory indices o[k] of the four taps nw, ne, sw, se and their bilinear weights
// (0 for a tap outside the node grid), the arithmetic of flow_sample at the node coordinates.  `cell` is -1 when no tap
// lies inside the grid (or the coordinates are not finite: u = v = 0, as for the dense flow).
struct NodeSample {
    int o[4];
    float w[4];
    unsigned inside;   // bit k: tap k lies inside the node grid
    int cell;
};

__device__ __forceinline__ NodeSample node_sample(const GridArgs &A, float xe, float ye)
{
    NodeSample s;
    s.cell = -1;
    s.inside = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) { s.o[k] = 0; s.w[k] = 0.0f; }
    const float ix = __fmul_rn(xe, A.rx), iy = __fmul_rn(ye, A.ry);
    if (!(fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f)) return s;
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float xs = fx + 1.0f, ys = fy + 1.0f;
    const float w[4] = {__fmul_rn(__fsub_rn(xs, ix), __fsub_rn(ys, iy)), __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(ys, iy)),
                        __fmul_rn(__fsub_rn(xs, ix), __fsub_rn(iy, fy)), __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy))};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
        if ((unsigned)xx < (unsigned)A.gw && (unsigned)yy < (unsigned)A.gh) {
            s.o[k] = yy * A.gw + xx;
            s.w[k] = w[k];
            s.inside |= 1u << k;
        }
    }
    if (s.inside) s.cell = (y0 + 1) * (A.gw + 1) + (x0 + 1);   // x0, y0 >= -1 when a tap is inside
    return s;
}

// the flow of one candidate's nodes at an event, in flow_sample's order of terms (a tap outside the grid reads 0)
__device__ __forceinline__ void node_flow(const float2 *nodes, const NodeSample &s, float &u, float &v)
{
    u = 0.0f; v = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 q = s.inside >> k & 1u ? nodes[s.o[k]] : make_float2(0.0f, 0.0f);
        u = __fadd_rn(u, __fmul_rn(q.x, s.w[k]));
        v = __fadd_rn(v, __fmul_rn(q.y, s.w[k]));
    }
}

// the J grids of sample b, [J][2][gh][gw] in global memory, as [J][gh gw] {u, v} pairs in shared memory
__device__ __forceinline__ void load_nodes(const GridArgs &A, int b, float2 *nodes)
{
    const int G = A.gh * A.gw, J = A.J;
    const float *src = A.grid + (int64_t)b * J * 2 * G;
    for (int q = threadIdx.x; q < J * G; q += kFlowObjThreads) {
        const int j = q / G, k = q - j * G;
        nodes[q] = make_float2(__ldg(src + (2 * j) * G + k), __ldg(src + (2 * j + 1) * G + k));
    }
    __syncthreads();
}

// the record of one event that a grid-flow pass reads: 16 bytes for the contrast loss, 20 for the timestamp loss (TS)
template <bool TS>
__device__ __forceinline__ auto load_grid_event(const EventSource &E, int64_t i)
{
    if constexpr (TS) return load_xytup(E, i);
    else return load_xytp(E, i);
}

template <bool TS>
__global__ void __launch_bounds__(kFlowObjThreads) grid_flow_cand_kernel(const GridArgs A)
{
    extern __shared__ float2 grid_nodes[];   // [J][gh gw]
    const int b = blockIdx.y, J = A.J, G = A.gh * A.gw;
    load_nodes(A, b, grid_nodes);
    int64_t first, last;
    sample_range(A.F.E, b, first, last);
    const int Wc = A.F.C.Wc;
    const int64_t npix = (int64_t)A.F.C.Hc * Wc;
    float *acc = A.F.acc + (int64_t)b * J * npix * (TS ? 2 * 8 : 4);   // per canvas: one IWE block or two {S, C} blocks
    unsigned nonfinite = 0;   // bit j: candidate j warped an event to a non-finite position (J <= 32)
    for_each_event(first, last, [&](int64_t i) { return load_grid_event<TS>(A.F.E, i); }, [&](int64_t, const auto &e) {
        const NodeSample s = node_sample(A, e.x, e.y);
        for (int j = 0; j < J; ++j) {
            float u, v;
            node_flow(grid_nodes + j * G, s, u, v);
            Taps T;
            bool nf = false;
            if constexpr (TS) {
                // weight 1; a NaN p is dropped after the non-finite check, as in flow_ts_event
                const int pol = ts_polarity(e.p);
                if (flow_obj_keep(A.F, e.x, e.y, u, v, e.t, 1.0f, T, nf) && pol >= 0)
                    ts_block_add(acc + (int64_t)j * 2 * npix * 8, npix, Wc, pol, T, e.tau);
            } else if (flow_obj_keep(A.F, e.x, e.y, u, v, e.t, e.p, T, nf)) {
                red_add4(acc + ((int64_t)j * npix + (int64_t)T.y0 * Wc + T.x0) * 4, T.ti);
            }
            if (nf) nonfinite |= 1u << j;
        }
    });
    for (int j = 0; j < J; ++j)
        if (nonfinite >> j & 1u) A.F.nonfinite[(int64_t)b * J + j] = 1u;
}

// v[0..N-1] summed over the lanes of the warp that share `key` (all 32 lanes call this); the lowest lane of each key
// holds the sum and gets true.  A shuffle tree over each key's peers (the lanes of rank 2^r k add the next peer's partial
// sum).
template <int N>
__device__ __forceinline__ bool warp_key_sum(int key, float (&v)[N])
{
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(full, key);
    unsigned rank = __popc(peers & ((1u << lane) - 1u));
    unsigned rest = peers & (0xfffffffeu << lane);   // the peers above this lane
    while (__any_sync(full, rest != 0u)) {
        const int next = __ffs(rest);
        float t[N];
#pragma unroll
        for (int k = 0; k < N; ++k) t[k] = __shfl_sync(full, v[k], (next - 1) & 31);
        if (next) {
#pragma unroll
            for (int k = 0; k < N; ++k) v[k] += t[k];
        }
        rest &= __ballot_sync(full, !(rank & 1u));
        rank >>= 1;
    }
    return lane == __ffs(peers) - 1;
}

// One event's node terms: (gu, gv) = df/d(u, v) times the four node weights of s into val (u taps, then v taps), keyed
// by the node cell.  Untouched when both are zero.
__device__ __forceinline__ void node_terms(const NodeSample &s, float gu, float gv, float (&val)[8], int &key)
{
    if (gu != 0.0f || gv != 0.0f) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (s.inside >> q & 1u) { val[q] = gu * s.w[q]; val[4 + q] = gv * s.w[q]; }
        }
        key = s.cell;
    }
}

// The depth grid's one-channel node_terms: g = df/drho times the four node weights of s into val, keyed by the node cell
__device__ __forceinline__ void node_terms(const NodeSample &s, float g, float (&val)[4], int &key)
{
    if (g != 0.0f) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (s.inside >> q & 1u) val[q] = g * s.w[q];
        }
        key = s.cell;
    }
}

// The terms of the lanes of the warp with the same key summed (warp_key_sum) and added by one lane per node cell to the
// CTA's f64 accumulator acc [NC][G] in shared memory (NC channels: 2 for the flow, 1 for the inverse depth; val holds
// the four taps of each channel in turn).  All 32 lanes call this; a lane without a term has its own key.
template <int NC>
__device__ __forceinline__ void node_grad_flush(double *acc, int G, const NodeSample &s, int key, float (&val)[4 * NC])
{
    if (warp_key_sum(key, val) && key >= 0) {
        // the peers share the leader's cell and so its taps inside the grid
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (!(s.inside >> q & 1u)) continue;
#pragma unroll
            for (int c = 0; c < NC; ++c)
                if (val[4 * c + q] != 0.0f) atomicAdd(acc + c * G + s.o[q], (double)val[4 * c + q]);
        }
    }
}

// The node-gradient pass of both grid-flow losses.  The event loop is written out rather than taken from a lambda-driven
// helper such as for_each_event: that form costs the contrast pass 3 registers.
template <bool TS>
__global__ void __launch_bounds__(kFlowObjThreads) grid_flow_grad_kernel(const GridArgs A)
{
    using Ev = decltype(load_grid_event<TS>(A.F.E, 0));
    extern __shared__ double grid_acc[];   // [2][gh gw] f64, then the nodes as [gh gw] {u, v}
    const int b = blockIdx.y, G = A.gh * A.gw;
    float2 *nodes = reinterpret_cast<float2 *>(grid_acc + 2 * G);
    for (int q = threadIdx.x; q < 2 * G; q += kFlowObjThreads) grid_acc[q] = 0.0;
    load_nodes(A, b, nodes);   // and the barrier
    int64_t first, last;
    sample_range(A.F.E, b, first, last);
    const int Wc = A.F.C.Wc;
    const int64_t npix = (int64_t)A.F.C.Hc * Wc;
    const float *Wb = TS ? nullptr : A.F.Wimg + b * npix;        // contrast: W_b
    const float2 *ab = TS ? A.F.ab + b * 2 * npix : nullptr;     // timestamp: the (A, B) pairs of both polarities
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * kFlowObjThreads;
    // warp-uniform trip count (warp_key_sum needs every lane): kBatch records per lane, masked past `last`
    for (int64_t i0 = first + (int64_t)blockIdx.x * kFlowObjThreads + (threadIdx.x - lane); i0 < last; i0 += kBatch * stride) {
        Ev ev[kBatch];
#pragma unroll
        for (int k = 0; k < kBatch; ++k) {
            const int64_t q = i0 + k * stride + lane;
            ev[k] = q < last ? load_grid_event<TS>(A.F.E, q) : Ev{};
            if (!(q < last)) ev[k].x = __int_as_float(0x7fc00000);   // a NaN position: no cell, no term
        }
#pragma unroll
        for (int k = 0; k < kBatch; ++k) {
            const Ev &e = ev[k];
            const NodeSample s = node_sample(A, e.x, e.y);
            float val[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) val[q] = 0.0f;
            int key = -1 - lane;   // a lane without a term is alone with its key
            float u, v;
            node_flow(nodes, s, u, v);
            Taps T;
            bool nf = false;
            if constexpr (TS) {
                // weight 1 and a NaN p dropped, as in flow_ts_event; dF/dk = tau A + B per tap of the event's polarity
                const int pol = ts_polarity(e.p);
                if (s.cell >= 0 && flow_obj_keep(A.F, e.x, e.y, u, v, e.t, 1.0f, T, nf) && pol >= 0) {
                    const float2 *abs_ = pol ? ab + npix : ab;
                    const float dx = T.dx, dy = T.dy;
                    const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
                    const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
                    const float2 a00 = __ldg(abs_ + r0 + T.x0), a01 = __ldg(abs_ + r0 + T.x1), a10 = __ldg(abs_ + r1 + T.x0),
                                 a11 = __ldg(abs_ + r1 + T.x1);
                    const float tau = e.tau;
                    const float q00 = tau * a00.x + a00.y, q01 = tau * a01.x + a01.y, q10 = tau * a10.x + a10.y,
                                q11 = tau * a11.x + a11.y;
                    float sx, sy;
                    tap_slopes(ox, oy, dx, dy, q00, q01, q10, q11, sx, sy);
                    node_terms(s, sx * e.t, sy * e.t, val, key);
                }
            } else if (s.cell >= 0 && flow_obj_keep(A.F, e.x, e.y, u, v, e.t, e.p, T, nf)) {
                // df/dx' and df/dy' through the four bilinear taps of the IWE, as in flow_obj_event
                const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
                const float w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0),
                            w11 = __ldg(Wb + r1 + T.x1);
                const float ox = 1.0f - T.dx, oy = 1.0f - T.dy;
                float sx, sy;
                tap_slopes(ox, oy, T.dx, T.dy, w00, w01, w10, w11, sx, sy);
                node_terms(s, T.wm * sx * e.t, T.wm * sy * e.t, val, key);
            }
            node_grad_flush<2>(grid_acc, G, s, key, val);
        }
    }
    __syncthreads();
    double *dst = A.grad + (int64_t)b * 2 * G;
    for (int q = threadIdx.x; q < 2 * G; q += kFlowObjThreads)
        if (grid_acc[q] != 0.0) atomicAdd(dst + q, grid_acc[q]);
}

// [B][2][gh][gw] f64 sums -> the f32 gradient
__global__ void __launch_bounds__(256) grid_flow_grad_cast_kernel(const double *__restrict__ g, float *__restrict__ out, int64_t n)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (float)g[i];
}

// Shared argument checks and set-up of the grid-flow entries.  n_cand 0: the differentiable entries (one canvas per
// sample, gh gw <= kMaxGridNodes); else n_cand forward-only canvases per sample (n_cand <= kMaxCandidates,
// n_cand gh gw <= kMaxGridCandNodes).  `images` tail images per canvas (1 for the contrast loss, 2 for the timestamp loss,
// one per polarity), and at most 65535 images: batch (n_cand) <= 65535 / images.
static int grid_flow_limits(int batch, int n_cand, int gh, int gw, int H, int W, int images = 1)
{
    if (batch < 0 || !batch_canvas_ok(H, W) || gh < 2 || gw < 2 || gh > H || gw > W) return 0;
    const int64_t G = (int64_t)gh * gw, canvases = 65535 / images;
    if (!n_cand) return batch <= canvases && G <= kMaxGridNodes;
    return n_cand >= 1 && n_cand <= kMaxCandidates && (int64_t)n_cand * G <= kMaxGridCandNodes && (int64_t)batch * n_cand <= canvases;
}

// tau: the timestamp loss's normalised stamps (images 2, with its objective OBJ_SOS and acc_blocks flow_ts_acc_blocks);
// acc_blocks: 16-byte accumulator blocks per image (batch_obj_carve)
static int grid_flow_setup(const char *who, const float *x, const float *y, const float *t, const float *tau, const float *p,
                           const int64_t *offsets, int batch, int64_t n, const float *grid, int n_cand, int gh, int gw, int H, int W,
                           double sigma, int objective, int images, size_t acc_blocks, void *workspace, size_t workspace_bytes,
                           GridArgs &A, BatchObjWorkspace &ws, BlurTaps &taps, const char *wrt = "flow")
{
    if (int rc = check_sigma(who, sigma)) return rc;
    if (!grid_flow_limits(batch, n_cand, gh, gw, H, W, images) || n < 0 || (batch > 0 && (!offsets || !grid)) ||
        (n > 0 && (!x || !y || !t || (images == 2 && !tau) || !p))) {
        set_error("%s: bad arguments (2 <= gh <= H, 2 <= gw <= W, gh gw <= %d; candidates: 1 <= n_cand <= %d, n_cand gh gw "
                  "<= %d, batch n_cand <= %d; else batch <= %d)", who, kMaxGridNodes, kMaxCandidates, kMaxGridCandNodes,
                  65535 / images, 65535 / images);
        return EVK_E_ARG;
    }
    const int J = n_cand ? n_cand : 1;
    int rc = batch_obj_check(who, wrt, images * batch * J, H, W, sigma, objective, acc_blocks, workspace, workspace_bytes, ws,
                             taps, !n_cand);
    if (rc) return rc;
    A = GridArgs{};
    A.F.C.Hc = H + 1; A.F.C.Wc = W + 1;
    A.F.E = EventSource{x, y, t, p, tau, offsets, n};
    A.F.H = H; A.F.W = W;
    A.F.acc = ws.acc;
    A.F.nonfinite = ws.nonfinite;
    A.grid = grid;
    A.gh = gh; A.gw = gw; A.J = J;
    A.rx = (float)(gw - 1) / (float)(W - 1);
    A.ry = (float)(gh - 1) / (float)(H - 1);
    return EVK_OK;
}

// forward and candidates, before the tail: zero the counters and the accumulators of the batch J canvases, the event pass
template <bool TS>
static int grid_flow_event_pass(const GridArgs &A, const BatchObjWorkspace &ws, int batch, cudaStream_t st)
{
    const int npix = A.F.C.Hc * A.F.C.Wc, canvases = batch * A.J;
    EVK_CUDA(batch_obj_zero(ws, (TS ? 2 : 1) * (int64_t)canvases, npix, TS ? 8 : 4, st));
    if (A.F.E.n > 0) {
        const size_t smem = (size_t)A.J * A.gh * A.gw * sizeof(float2);
        EVK_CUDA(cudaFuncSetAttribute(grid_flow_cand_kernel<TS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ProfScope prof(st);
        prof_count(1);
        grid_flow_cand_kernel<TS><<<batch_grid(A.F.E.n, batch), kFlowObjThreads, smem, st>>>(A);
    }
    return EVK_OK;
}

// forward and candidates of the contrast loss: the event pass, the tail into iwe_out (the candidates: ws.Wimg)
static int grid_flow_forward(const GridArgs &A, const BatchObjWorkspace &ws, const BlurTaps &taps, int batch, int objective,
                             double obj_param, float *iwe_out, double *f_out, cudaStream_t st)
{
    if (int rc = grid_flow_event_pass<false>(A, ws, batch, st)) return rc;
    batch_obj_forward_tail(ws, A.F.C.Hc, A.F.C.Wc, taps, batch * A.J, objective, obj_param, iwe_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// backward, after the image-space half (which set A.F.Wimg or A.F.ab): the node pass into the f64 sums A.grad (zeroed by
// the caller), then their cast to grad_grid
template <bool TS>
static int grid_flow_node_grad(const GridArgs &A, int batch, float *grad_grid, cudaStream_t st)
{
    const int64_t nodes = (int64_t)batch * 2 * A.gh * A.gw;
    if (A.F.E.n > 0) {
        const size_t smem = (size_t)A.gh * A.gw * (2 * sizeof(double) + sizeof(float2));
        EVK_CUDA(cudaFuncSetAttribute(grid_flow_grad_kernel<TS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ProfScope prof(st);
        prof_count(1);
        grid_flow_grad_kernel<TS><<<batch_grid(A.F.E.n, batch), kFlowObjThreads, smem, st>>>(A);
    }
    prof_count(1);
    grid_flow_grad_cast_kernel<<<grid_simple(nodes, 256), 256, 0, st>>>(A.grad, grad_grid, nodes);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// ---- depth from a known camera motion: an inverse-depth node grid per sample (evk_cmax_depth_grid_*) ---------------
// The camera-motion contrast objective (model_taps<WARP_CAMERA_MOTION_F32>) with each event's rho interpolated from a
// gh x gw grid of inverse-depth nodes of its sample instead of read from memory: node_sample and node_flow's arithmetic
// with one channel (a tap outside the grid reads 0), then the camera motion's keep rules, warp, bounds mask and splat,
// and the contrast loss's image tail.  The motion rows (wx, wy, wz, vx, vy, vz, fx, fy) are data; only the nodes get a
// gradient.  The grid of both event passes is (slices, batch), and every CTA holds its sample's nodes in dynamic shared
// memory as f32:
//   forward / candidates: depth_grid_cand_kernel.  Per event one 16-byte record, the node cell and its weights once and
//             the rotation U = exp([theta]x) b once (cam_rotate: it depends on neither rho nor the candidate), then per
//             candidate j the interpolated rho, P = U + (rho d) v, the projection, the keep rules and one v4 reduction into
//             canvas z = b J + j, scored by batch_obj_forward_tail.
//   backward: batch_obj_backward_W, then depth_grid_grad_kernel: per event the four gathers of W_b give df/dx', df/dy',
//             times dx'/drho = d fx iz (vx - X vz) and dy'/drho = d fy iz (vy - Y vz) and the four node weights; the
//             lanes of a warp with the same node cell sum their four values (warp_key_sum), one lane per cell adds them to
//             a per-CTA f64 accumulator [gh][gw] in shared memory, and one f64 atomic per node and CTA goes to
//             [B][gh][gw] in the workspace, cast to the f32 output by grid_flow_grad_cast_kernel.
// The limits are the grid flow's (grid_flow_limits): gh gw <= kMaxGridNodes for the loss and n_cand gh gw <=
// kMaxGridCandNodes for the candidates -- half the grid flow's shared memory, since a node is one float.
// The depth-grid average-timestamp loss (evk_depth_grid_timestamp_*) runs the same passes with TS = true: a 20-byte
// record per event, weight 1, the two v4 reductions of ts_block_add into image pair z = 2 (b J + j) + s and
// ts_obj_forward_tail; a non-finite warp contributes nothing and flags no sample (motion_ts_event_kernel's rule).  Its
// backward gathers the (A, B) pairs of ts_obj_backward_ab instead of W_b, as grid_flow_grad_kernel<true> does, and
// contracts df/dx', df/dy' with the same dx'/drho, dy'/drho, without the splat weight.
struct DepthGridArgs {
    GridArgs G;             // canvas and bounds mask (F.C), events, nodes [B][J][gh][gw], accumulators, node sums
    const double *motion;   // [B][8] rows (wx, wy, wz, vx, vy, vz, fx, fy); the joint candidates: [B][J][8]
    double cx, cy;          // the principal point
    double *grad_motion;    // the joint backward: [B][6]
};

// a camera motion as model_taps reads it: every value rounded to f32
struct CamMotion {
    float wx, wy, wz, vx, vy, vz, fx, fy, cx, cy;
};
__device__ __forceinline__ CamMotion cam_motion_row(const double *m, double cx, double cy)
{
    return {(float)m[0], (float)m[1], (float)m[2], (float)m[3], (float)m[4], (float)m[5], (float)m[6], (float)m[7],
            (float)cx, (float)cy};
}
// sample b's camera motion
__device__ __forceinline__ CamMotion cam_motion(const DepthGridArgs &D, int b)
{
    return cam_motion_row(D.motion + (int64_t)b * 8, D.cx, D.cy);
}

// the J inverse-depth grids of sample b, [J][gh gw] floats, into shared memory
__device__ __forceinline__ void load_depth_nodes(const GridArgs &A, int b, float *nodes)
{
    const int n = A.J * A.gh * A.gw;
    const float *src = A.grid + (int64_t)b * n;
    for (int q = threadIdx.x; q < n; q += kFlowObjThreads) nodes[q] = __ldg(src + q);
    __syncthreads();
}

// one candidate's inverse depth at an event: node_flow with one channel
__device__ __forceinline__ float node_depth(const float *nodes, const NodeSample &s)
{
    float r = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k) r = __fadd_rn(r, __fmul_rn(s.inside >> k & 1u ? nodes[s.o[k]] : 0.0f, s.w[k]));
    return r;
}

// The camera motion's warp of one event at inverse depth rho, from its rotation r: the keep rules of model_taps (a
// negative or non-finite rho, Pz <= 0 or a non-finite Pz, the bounds mask) and the taps.  q: the projection.
__device__ __forceinline__ bool depth_taps(const CmaxArgs &C, const CamMotion &m, const CamRot &r, float rho, float d, float p,
                                           CamProj &q, Taps &T)
{
    if (!(rho >= 0.0f) || isinf(rho)) return false;
    if (!cam_project<true>(r, rho * d, m.vx, m.vy, m.vz, q)) return false;
    unsigned oob = 0;   // a kept finite event lies inside the canvas; a non-finite one contributes nothing
    return model_keep_taps(C, q.xw, q.yw, p, oob, T);
}

// JOINT: the joint candidates pass (evk_cmax_depth_grid_joint_candidates_f32), whose candidate j is the pair (motion
// row [b][j], grid [b][j]): the J motions sit behind the J grids in shared memory, and the rotation is per candidate.
template <bool TS, bool JOINT = false>
__global__ void __launch_bounds__(kFlowObjThreads) depth_grid_cand_kernel(const DepthGridArgs D)
{
    extern __shared__ float depth_nodes[];   // [J][gh gw], then JOINT: CamMotion [J]
    const GridArgs &A = D.G;
    const int b = blockIdx.y, J = A.J, G = A.gh * A.gw;
    CamMotion *motions = reinterpret_cast<CamMotion *>(depth_nodes + J * G);
    if constexpr (JOINT) {
        for (int j = threadIdx.x; j < J; j += kFlowObjThreads)
            motions[j] = cam_motion_row(D.motion + ((int64_t)b * J + j) * 8, D.cx, D.cy);
    }
    load_depth_nodes(A, b, depth_nodes);   // and the barrier
    int64_t first, last;
    sample_range(A.F.E, b, first, last);
    const CmaxArgs &C = A.F.C;
    const int64_t npix = (int64_t)C.Hc * C.Wc;
    float *acc = A.F.acc + (int64_t)b * J * npix * (TS ? 2 * 8 : 4);   // per canvas: one IWE block or two {S, C} blocks
    const CamMotion m = JOINT ? CamMotion{} : cam_motion(D, b);
    for_each_event(first, last, [&](int64_t i) { return load_grid_event<TS>(A.F.E, i); }, [&](int64_t, const auto &e) {
        const int pol = TS ? ts_polarity(e.p) : 0;
        if (pol < 0) return;   // a NaN p is in neither timestamp image
        const NodeSample s = node_sample(A, e.x, e.y);
        CamRot r;
        if constexpr (!JOINT) r = cam_rotate(e.x, e.y, e.t, m.wx, m.wy, m.wz, m.fx, m.fy, m.cx, m.cy);
        for (int j = 0; j < J; ++j) {
            CamProj q;
            Taps T;
            const CamMotion &mj = JOINT ? motions[j] : m;
            if constexpr (JOINT) r = cam_rotate(e.x, e.y, e.t, mj.wx, mj.wy, mj.wz, mj.fx, mj.fy, mj.cx, mj.cy);
            if constexpr (TS) {
                if (depth_taps(C, mj, r, node_depth(depth_nodes + j * G, s), e.t, 1.0f, q, T))
                    ts_block_add(acc + (int64_t)j * 2 * npix * 8, npix, C.Wc, pol, T, e.tau);
            } else if (depth_taps(C, mj, r, node_depth(depth_nodes + j * G, s), e.t, e.p, q, T)) {
                red_add4(acc + ((int64_t)j * npix + (int64_t)T.y0 * C.Wc + T.x0) * 4, T.ti);
            }
        }
    });
}

// The node-gradient pass of both depth-grid losses, written out like grid_flow_grad_kernel (warp_key_sum needs every
// lane).  MOTION: the joint backward (evk_cmax_depth_grid_joint_grad_f32), which also contracts df/dx', df/dy' with the
// camera motion's Jacobian rows at the event's rho (cam_jacobian), in f64 as motion_obj_event_kernel does, into six
// per-thread sums that one CTA reduction and one f64 atomic per component and CTA add to grad_motion [B][6].
template <bool TS, bool MOTION = false>
__global__ void __launch_bounds__(kFlowObjThreads) depth_grid_grad_kernel(const DepthGridArgs D)
{
    static_assert(!(TS && MOTION), "the average-timestamp loss has no joint backward");
    using Ev = decltype(load_grid_event<TS>(D.G.F.E, 0));
    extern __shared__ double depth_acc[];   // [gh gw] f64, then the nodes [gh gw] f32
    const GridArgs &A = D.G;
    const int b = blockIdx.y, G = A.gh * A.gw;
    float *nodes = reinterpret_cast<float *>(depth_acc + G);
    for (int q = threadIdx.x; q < G; q += kFlowObjThreads) depth_acc[q] = 0.0;
    load_depth_nodes(A, b, nodes);   // and the barrier
    int64_t first, last;
    sample_range(A.F.E, b, first, last);
    const CmaxArgs &C = A.F.C;
    const int Wc = C.Wc;
    const int64_t npix = (int64_t)C.Hc * Wc;
    const float *Wb = TS ? nullptr : A.F.Wimg + b * npix;        // contrast: W_b
    const float2 *ab = TS ? A.F.ab + b * 2 * npix : nullptr;     // timestamp: the (A, B) pairs of both polarities
    const CamMotion m = cam_motion(D, b);
    double u[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) u[k] = 0.0;
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * kFlowObjThreads;
    for (int64_t i0 = first + (int64_t)blockIdx.x * kFlowObjThreads + (threadIdx.x - lane); i0 < last; i0 += kBatch * stride) {
        Ev ev[kBatch];
#pragma unroll
        for (int k = 0; k < kBatch; ++k) {
            const int64_t q = i0 + k * stride + lane;
            ev[k] = q < last ? load_grid_event<TS>(A.F.E, q) : Ev{};
            if (!(q < last)) ev[k].x = __int_as_float(0x7fc00000);   // a NaN position: no cell, no term
        }
#pragma unroll
        for (int k = 0; k < kBatch; ++k) {
            const Ev &e = ev[k];
            const NodeSample s = node_sample(A, e.x, e.y);
            float val[4] = {0.0f, 0.0f, 0.0f, 0.0f};
            int key = -1 - lane;   // a lane without a term is alone with its key
            const int pol = TS ? ts_polarity(e.p) : 0;   // a NaN p: no term
            // an event with no node cell (beyond the grid's outer nodes, or the NaN padding) has rho = 0 and no node
            // term, but where its taps are kept it counts in f and depends on the motion, as in the forward
            if ((MOTION || s.cell >= 0) && pol >= 0) {
                const CamRot r = cam_rotate(e.x, e.y, e.t, m.wx, m.wy, m.wz, m.fx, m.fy, m.cx, m.cy);
                CamProj q;
                Taps T;
                const float rho = node_depth(nodes, s);
                const bool kept = depth_taps(C, m, r, rho, e.t, TS ? 1.0f : e.p, q, T);
                if (kept && (!MOTION || s.cell >= 0)) {
                    float sx, sy;
                    if constexpr (TS) {
                        // dF/dk = tau A + B per tap of the event's polarity, as in grid_flow_grad_kernel<true>
                        const float2 *abs_ = pol ? ab + npix : ab;
                        const float dx = T.dx, dy = T.dy;
                        const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
                        const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
                        const float2 a00 = __ldg(abs_ + r0 + T.x0), a01 = __ldg(abs_ + r0 + T.x1),
                                     a10 = __ldg(abs_ + r1 + T.x0), a11 = __ldg(abs_ + r1 + T.x1);
                        const float tau = e.tau;
                        const float q00 = tau * a00.x + a00.y, q01 = tau * a01.x + a01.y, q10 = tau * a10.x + a10.y,
                                    q11 = tau * a11.x + a11.y;
                        tap_slopes(ox, oy, dx, dy, q00, q01, q10, q11, sx, sy);
                    } else {
                        const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
                        const float w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0),
                                    w11 = __ldg(Wb + r1 + T.x1);
                        const float ox = 1.0f - T.dx, oy = 1.0f - T.dy;
                        tap_slopes(ox, oy, T.dx, T.dy, w00, w01, w10, w11, sx, sy);
                    }
                    const float di = e.t * q.iz;   // dx'/drho = d fx iz (vx - X vz), dy'/drho = d fy iz (vy - Y vz)
                    const float jx = (di * m.fx) * (m.vx - q.X * m.vz), jy = (di * m.fy) * (m.vy - q.Y * m.vz);
                    if constexpr (TS) node_terms(s, sx * jx + sy * jy, val, key);
                    else node_terms(s, T.wm * (sx * jx + sy * jy), val, key);
                }
                if constexpr (MOTION && !TS) {
                    if (kept) {
                        float mx[8], my[8];
                        cam_jacobian<true>(r, q, rho * e.t, e.t, mx, my);
                        const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
                        const double w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0),
                                     w11 = __ldg(Wb + r1 + T.x1);
                        const double dx = T.dx, dy = T.dy, ox = 1.0 - dx, oy = 1.0 - dy, wm = T.wm;
                        double dsx, dsy;
                        tap_slopes(ox, oy, dx, dy, w00, w01, w10, w11, dsx, dsy);
#pragma unroll
                        for (int k = 0; k < 6; ++k) u[k] += wm * ((double)mx[k] * dsx + (double)my[k] * dsy);
                    }
                }
            }
            node_grad_flush<1>(depth_acc, G, s, key, val);
        }
    }
    __syncthreads();
    double *dst = A.grad + (int64_t)b * G;
    for (int q = threadIdx.x; q < G; q += kFlowObjThreads)
        if (depth_acc[q] != 0.0) atomicAdd(dst + q, depth_acc[q]);
    if constexpr (MOTION) cta_add<6, kFlowObjThreads>(u, D.grad_motion + (int64_t)b * 6);
}

// The checks and set-up of the depth-grid entries: grid_flow_setup's, then the motion rows.  `images` per canvas: 1 for
// the contrast loss, 2 for the timestamp loss (with its stamps tau, objective OBJ_SOS and acc_blocks flow_ts_acc_blocks).
static int depth_grid_setup(const char *who, const float *x, const float *y, const float *t, const float *tau, const float *p,
                            const int64_t *offsets, int batch, int64_t n, const double *motion, double cx, double cy,
                            const float *grid, int n_cand, int gh, int gw, int H, int W, double sigma, int objective,
                            int images, void *workspace, size_t workspace_bytes, DepthGridArgs &D, BatchObjWorkspace &ws,
                            BlurTaps &taps)
{
    const size_t acc_blocks = images == 2 ? flow_ts_acc_blocks(H, W) : (size_t)(H + 1) * (W + 1);
    int rc = grid_flow_setup(who, x, y, t, tau, p, offsets, batch, n, grid, n_cand, gh, gw, H, W, sigma, objective, images,
                             acc_blocks, workspace, workspace_bytes, D.G, ws, taps, "inverse depth");
    if (rc) return rc;
    if (batch > 0 && !motion) { set_error("%s: null motion", who); return EVK_E_ARG; }
    D.G.F.C.Hm = H; D.G.F.C.Wm = W;
    D.G.F.C.p_scale = 1.0;
    D.motion = motion;
    D.cx = cx; D.cy = cy;
    D.grad_motion = nullptr;
    return EVK_OK;
}

// forward and candidates, before the tail: zero the counters and the accumulators of the batch J canvases, the event
// pass.  nonfinite stays zero: a non-finite event contributes nothing (model_taps).  JOINT: one motion per candidate.
template <bool TS, bool JOINT = false>
static int depth_grid_event_pass(const DepthGridArgs &D, const BatchObjWorkspace &ws, int batch, cudaStream_t st)
{
    const GridArgs &A = D.G;
    const int npix = A.F.C.Hc * A.F.C.Wc, canvases = batch * A.J;
    EVK_CUDA(batch_obj_zero(ws, (TS ? 2 : 1) * (int64_t)canvases, npix, TS ? 8 : 4, st));
    if (A.F.E.n > 0) {
        const size_t smem = (size_t)A.J * A.gh * A.gw * sizeof(float) + (JOINT ? A.J * sizeof(CamMotion) : 0);
        EVK_CUDA(cudaFuncSetAttribute(depth_grid_cand_kernel<TS, JOINT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
        ProfScope prof(st);
        prof_count(1);
        depth_grid_cand_kernel<TS, JOINT><<<batch_grid(A.F.E.n, batch), kFlowObjThreads, smem, st>>>(D);
    }
    return EVK_OK;
}

// forward and candidates of the contrast loss: the event pass, the tail into iwe_out (the candidates: ws.Wimg)
template <bool JOINT = false>
static int depth_grid_forward(const DepthGridArgs &D, const BatchObjWorkspace &ws, const BlurTaps &taps, int batch,
                              int objective, double obj_param, float *iwe_out, double *f_out, cudaStream_t st)
{
    if (int rc = depth_grid_event_pass<false, JOINT>(D, ws, batch, st)) return rc;
    batch_obj_forward_tail(ws, D.G.F.C.Hc, D.G.F.C.Wc, taps, batch * D.G.J, objective, obj_param, iwe_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// backward, after the image-space half (which set D.G.F.Wimg or D.G.F.ab): the node pass into the f64 sums D.G.grad
// (zeroed by the caller), then their cast to grad_grid.  MOTION: also the motion gradient into D.grad_motion (zeroed
// by the caller).
template <bool TS, bool MOTION = false>
static int depth_grid_node_grad(const DepthGridArgs &D, int batch, float *grad_grid, cudaStream_t st)
{
    const GridArgs &A = D.G;
    const int64_t G = (int64_t)A.gh * A.gw, nodes = batch * G;
    if (A.F.E.n > 0) {
        const size_t smem = (size_t)G * (sizeof(double) + sizeof(float));
        EVK_CUDA(cudaFuncSetAttribute(depth_grid_grad_kernel<TS, MOTION>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
        ProfScope prof(st);
        prof_count(1);
        depth_grid_grad_kernel<TS, MOTION><<<batch_grid(A.F.E.n, batch), kFlowObjThreads, smem, st>>>(D);
    }
    prof_count(1);
    grid_flow_grad_cast_kernel<<<grid_simple(nodes, 256), 256, 0, st>>>(A.grad, grad_grid, nodes);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

// ---- parametric motion objective over a batch of samples (evk_cmax_motion_objective_f32 / _grad_f32) ---------------
// Sample b = events [offsets[b], offsets[b+1]) (clipped to [0, n)) warped by its own model params[b] -- linvel, rotation,
// xyztheta, affine, homography or camera rotation through model_taps, with the bounds mask of event_util.py:26-27 at img_size = (H, W) and the splat of
// image.py:179-217 on the (H+1)x(W+1) canvas -- then blurred and scored by the flow objective's image-space tail.  The
// grid of both event passes is (slices, batch), as for the flow objective:
//   forward:  one v4 reduction per kept event into the sample's 2x2-block image [B][Hc][Wc][4] (16 B per pixel)
//   backward: W_b = G(g_b C_b) per sample (batch_obj_backward_W), then per event the four taps of W_b (L2 gathers) against
//             the event's Jacobian (model_taps<..., true>), summed in f64 per thread as cmax_grad_pass_kernel does; a CTA
//             reduction and one f64 atomic per component and CTA into grad [B][K] -- no reduction per event, and no
//             canvas-size limit (W is not held in shared memory).
struct ModelArgs {
    CmaxArgs C;              // canvas (Hc, Wc) and bounds mask (Hm, Wm) for model_taps; p_scale 1, t_ref 0
    EventSource E;
    const double *params;    // [B][M][J][K] on the device (M models per sample when segmenting, J candidates per model)
    double cx, cy;           // the centre of xyztheta and the planar models, the camera rotation's principal point
    int M, J;
    float *acc;              // forward: the canvases' blocks
    const float *Wimg;       // contrast backward: W of every canvas [B][M][Hc][Wc]
    const float2 *ab;        // timestamp backward: (A, B) [B][2][Hc][Wc]
    double *grad;            // backward: [B][M][K]
    // segmentation
    const float *weights;    // [n][M]
    int wvec4;               // the weight rows load as float4s (M a multiple of 4, 16-byte aligned)
    const float *grad_f;     // backward: [B][M]
    const double *gsums;     // backward with the variance: the stats of every G_bm (sum(G) in [4])
    float *grad_w;           // backward: [n][M] or null
    const float *G;          // assignment: [B][M][Hc][Wc]
    double eps;              // assignment
    float *w_out;            // assignment: [n][M]
};

template <int WARP, bool GRAD>
__global__ void __launch_bounds__(kFlowObjThreads) motion_obj_event_kernel(const ModelArgs A)
{
    constexpr int K = model_dims(WARP);
    const int b = blockIdx.y;
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int64_t npix = (int64_t)A.C.Hc * A.C.Wc;
    ModelOf<WARP> M;
    load_model<WARP>(A.params, b, A.cx, A.cy, M);
    float *acc = GRAD ? nullptr : A.acc + b * npix * 4;
    const float *Wb = GRAD ? A.Wimg + b * npix : nullptr;
    double u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = 0.0;
    unsigned oob = 0;   // a kept finite event lies inside the canvas; a non-finite one contributes nothing
    auto load = [&](int64_t i) { return with_depth<WARP>(A.E, i, load_xytp(A.E, i)); };
    for_each_event(first, last, load, [&](int64_t, const Depthed<EvXYTP, has_depth(WARP)> &e) {
        Taps T;
        float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
        if (!model_taps<WARP, GRAD>(A.C, model_event<WARP>(e.x, e.y, e.t, e.p, depth_of(e)), M, oob, T, jx, jy)) return;
        if (!GRAD) {
            red_add4(acc + ((int64_t)T.y0 * A.C.Wc + T.x0) * 4, T.ti);
            return;
        }
        const int64_t r0 = (int64_t)T.y0 * A.C.Wc, r1 = (int64_t)T.y1 * A.C.Wc;
        const double w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0), w11 = __ldg(Wb + r1 + T.x1);
        const double dx = T.dx, dy = T.dy, ox = 1.0 - dx, oy = 1.0 - dy, wm = T.wm;
        double sx, sy;
        tap_slopes(ox, oy, dx, dy, w00, w01, w10, w11, sx, sy);
#pragma unroll
        for (int k = 0; k < K; ++k) u[k] += wm * ((double)jx[k] * sx + (double)jy[k] * sy);
    });
    if (GRAD) cta_add<K, kFlowObjThreads>(u, A.grad + (int64_t)b * K);
}

static int motion_obj_dims(int warp)
{
    switch (warp) {
    case EVK_WARP_LINVEL: return 2;
    case EVK_WARP_ROTATION: return 3;
    case EVK_WARP_XYZTHETA: return 4;
    case EVK_WARP_AFFINE: return 6;
    case EVK_WARP_HOMOGRAPHY: return 8;
    case EVK_WARP_CAMERA_ROTATION: return 5;
    default: return 0;
    }
}

// Shared argument checks and set-up of the model entries.  `images` per sample: 1 for the contrast losses, 2 for the
// timestamp losses (one per polarity; they also need tau), so that the tail's 65535 images allow 65535 or 32767 samples.
// n_cand 0: the differentiable entries, one set of images per sample; else a forward-only set per sample and candidate.
// acc_blocks: 16-byte accumulator blocks per image (batch_obj_carve).  depth: the entries with the inverse depth rho of
// every event, which take EVK_WARP_CAMERA_MOTION (K = 8) and nothing else; the other entries pass a null rho.
static int model_setup(const char *who, const float *x, const float *y, const float *t, const float *tau, const float *p,
                       const float *rho, bool depth, const int64_t *offsets, int batch, int64_t n, int warp,
                       const double *params, int K, double cx, double cy, int H, int W, double sigma, int objective,
                       int images, size_t acc_blocks, int n_cand, void *workspace, size_t workspace_bytes, ModelArgs &A,
                       BatchObjWorkspace &ws, BlurTaps &taps)
{
    if (int rc = check_sigma(who, sigma)) return rc;
    const int max_batch = 65535 / images;
    if (!batch_limits(batch, 0, H, W, images) || n < 0 || (batch > 0 && (!offsets || !params)) ||
        (n > 0 && (!x || !y || !t || (images == 2 && !tau) || !p || (depth && !rho)))) {
        set_error("%s: bad arguments (0 <= batch <= %d, H, W >= 2, (H+1)(W+1) <= 2^30)", who, max_batch);
        return EVK_E_ARG;
    }
    const int dims = depth ? (warp == EVK_WARP_CAMERA_MOTION ? 8 : 0) : motion_obj_dims(warp);
    if (!dims && depth) {
        set_error("%s: warp %d takes no inverse depth (only EVK_WARP_CAMERA_MOTION, %d)", who, warp, EVK_WARP_CAMERA_MOTION);
        return EVK_E_ARG;
    }
    if (!dims) { set_error("%s: unknown warp %d", who, warp); return EVK_E_ARG; }
    if (K != dims) { set_error("%s: warp %d has %d parameters, K = %d", who, warp, dims, K); return EVK_E_ARG; }
    if (n_cand && !batch_limits(batch, n_cand, H, W, images)) {
        set_error("%s: bad arguments (1 <= n_cand <= %d, batch * n_cand <= %d)", who, kMaxCandidates, max_batch);
        return EVK_E_ARG;
    }
    int rc = batch_obj_check(who, "parameters", images * batch * (n_cand ? n_cand : 1), H, W, sigma, objective, acc_blocks,
                             workspace, workspace_bytes, ws, taps, !n_cand);
    if (rc) return rc;
    A = ModelArgs{};
    A.C.Hm = H; A.C.Wm = W; A.C.Hc = H + 1; A.C.Wc = W + 1;
    A.C.p_scale = 1.0;
    A.E = EventSource{x, y, t, p, tau, offsets, n, rho};
    A.params = params; A.cx = cx; A.cy = cy;
    A.M = 1;
    A.J = n_cand ? n_cand : 1;
    A.acc = ws.acc;
    return EVK_OK;
}

// f(std::integral_constant<int, WARP>) for the f32 kernel WARP of a model warp (model_setup has checked it)
template <class F>
static void with_model_warp(int warp, F f)
{
    if (warp == EVK_WARP_LINVEL) f(std::integral_constant<int, WARP_LINVEL_F32>{});
    else if (warp == EVK_WARP_ROTATION) f(std::integral_constant<int, WARP_ROTATION_F32>{});
    else if (warp == EVK_WARP_AFFINE) f(std::integral_constant<int, WARP_AFFINE_F32>{});
    else if (warp == EVK_WARP_HOMOGRAPHY) f(std::integral_constant<int, WARP_HOMOGRAPHY_F32>{});
    else if (warp == EVK_WARP_CAMERA_ROTATION) f(std::integral_constant<int, WARP_CAMERA_ROTATION_F32>{});
    else f(std::integral_constant<int, WARP_XYZTHETA_F32>{});
}

// with_model_warp, and the camera motion for the entries with depth (the segmentation entries do not take it)
template <class F>
static void with_motion_warp(int warp, F f)
{
    if (warp == EVK_WARP_CAMERA_MOTION) f(std::integral_constant<int, WARP_CAMERA_MOTION_F32>{});
    else with_model_warp(warp, f);
}

// ---- motion segmentation by motion compensation (evk_cmax_motion_segment_*) ----------------------------------------
// Stoffregen, Gallego, Drummond, Kleeman, Scaramuzza (ICCV 2019): M motion models per sample and a soft membership
// w[e][m] of every event in every model.  Image (b, m) is the IWE of sample b's events warped by params[b][m], each
// event splatted with the f32 weight p_e w[e][m] through model_taps -- exactly the taps of the motion objective run on
// p * w[:, m] -- and canvas z = b M + m (candidates: (b M + m) J + j) goes through the same image tail.
//   forward / candidates: motion_seg_cand_kernel on the (slices, batch) grid, the sample's M x J models in shared
//             memory; each event is read once (16 B and its row of M weights) and costs one v4 reduction per kept
//             event and model / candidate.  Its unweighted instantiation (M = 1, no weight rows, splat weight p) is the
//             event pass of evk_cmax_motion_candidates_f32: n_cand parameter vectors of every sample (the grid search of
//             grid_search_initial, events_cmax.py:241-311, and the line search of a batched quasi-Newton fit), canvas
//             z = b n_cand + j, scored by batch_obj_forward_tail as the samples of evk_cmax_motion_objective_f32.
//   backward: motion_seg_grad_kernel on (slices, batch, M): per event the unweighted taps of model m (so that an event
//             of weight 0 still has its footprint), four gathers of W_bm, the parameter gradient of
//             motion_obj_event_kernel<.., true> with wm = p w[e][m], and optionally dF/dw[e][m] = p sum_taps k W_bm.
//   assignment (E-step): motion_seg_assign_kernel, per event and model c = max(0, sum_taps k G_bm) with the
//             polarity- and weight-free bilinear fractions k, then w'[e][m] = (c_m + eps) / (sum c + M eps).
constexpr int kMaxSegModels = 8;

__device__ __forceinline__ void load_seg_weights(const ModelArgs &A, int64_t i, float (&w)[kMaxSegModels])
{
    const float *r = A.weights + i * A.M;
    if (A.wvec4) {
#pragma unroll
        for (int q = 0; q < kMaxSegModels; q += 4) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q < A.M) v = ld_stream4(r + q);
            w[q] = v.x; w[q + 1] = v.y; w[q + 2] = v.z; w[q + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int m = 0; m < kMaxSegModels; ++m) w[m] = m < A.M ? ld_stream(r + m) : 0.0f;
    }
}

// what motion_seg_cand_kernel reads of an event: x, y, t, p, with DEPTH its inverse depth and, weighted, its row of M
// weights
template <bool DEPTH>
struct SegEvent {
    Depthed<EvXYTP, DEPTH> e;
    float w[kMaxSegModels];
};

// WEIGHTED: the segmentation's M x J models with the weight rows; else one model (M = 1) of J candidates, splat weight p
template <int WARP, bool WEIGHTED>
__global__ void __launch_bounds__(kFlowObjThreads) motion_seg_cand_kernel(const ModelArgs A)
{
    __shared__ ModelOf<WARP> mod[kMaxCandidates];
    const int b = blockIdx.y, M = WEIGHTED ? A.M : 1, J = A.J;
    load_models<WARP>(A.params, (int64_t)b * M * J, M * J, A.cx, A.cy, mod);
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int Wc = A.C.Wc;
    const int64_t npix = (int64_t)A.C.Hc * Wc;
    float *acc = A.acc + (int64_t)b * M * J * npix * 4;
    unsigned oob = 0;   // as in motion_obj_event_kernel: a kept finite event lies inside the canvas
    auto load = [&](int64_t q) {
        SegEvent<has_depth(WARP)> r;
        r.e = with_depth<WARP>(A.E, q, load_xytp(A.E, q));
        if (WEIGHTED) load_seg_weights(A, q, r.w);
        return r;
    };
    for_each_event_batch(first, last, load, [&](const SegEvent<has_depth(WARP)> (&e)[kBatch], int ne) {
#pragma unroll
        for (int m = 0; m < kMaxSegModels; ++m) {
            if (m >= M) break;
            for (int j = 0; j < J; ++j) {
                const ModelOf<WARP> Mo = mod[m * J + j];
                float *accq = acc + (int64_t)(m * J + j) * npix * 4;
#pragma unroll
                for (int k = 0; k < kBatch; ++k) {
                    if (k >= ne) continue;
                    const auto &ek = e[k].e;
                    const float p = WEIGHTED ? __fmul_rn(ek.p, e[k].w[m]) : ek.p;   // the splat weight p w, formed in f32
                    Taps T;
                    float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
                    if (model_taps<WARP, false>(A.C, model_event<WARP>(ek.x, ek.y, ek.t, p, depth_of(ek)), Mo, oob, T, jx, jy))
                        red_add4(accq + ((int64_t)T.y0 * Wc + T.x0) * 4, T.ti);
                }
            }
        }
    });
}

template <int WARP>
__global__ void __launch_bounds__(kFlowObjThreads) motion_seg_grad_kernel(const ModelArgs A)
{
    constexpr int K = model_dims(WARP);
    const int b = blockIdx.y, m = blockIdx.z, M = A.M;
    const int64_t z = (int64_t)b * M + m;
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int64_t npix = (int64_t)A.C.Hc * A.C.Wc;
    ModelOf<WARP> Mo;
    load_model<WARP>(A.params, z, A.cx, A.cy, Mo);
    const float *Wb = A.Wimg + z * npix;
    // W_bm leaves out the variance's constant -2 g mean(G) / P of dF/dI (the tap differences of the parameter gradient
    // cancel it, see flow_obj_coef_kernel); the weight gradient takes it back: dF/dI = W_bm + c0
    double c0 = 0.0;
    if (A.grad_w && A.gsums) c0 = 2.0 * (double)A.grad_f[z] * A.gsums[8 * z + 4] / ((double)npix * (double)npix);
    double u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = 0.0;
    unsigned oob = 0;
    const float *wcol = A.weights + m;
    auto load = [&](int64_t q) {
        const EvXYTP e = load_xytp(A.E, q);
        return EvXYTPW{e.x, e.y, e.t, e.p, __ldg(wcol + q * M)};
    };
    for_each_event(first, last, load, [&](int64_t i, const EvXYTPW &e) {
        Taps T;
        float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
        double gw = 0.0;
        // the footprint does not depend on the weight
        if (model_taps<WARP, true>(A.C, model_event<WARP>(e.x, e.y, e.t, 1.0f), Mo, oob, T, jx, jy)) {
            const int64_t r0 = (int64_t)T.y0 * A.C.Wc, r1 = (int64_t)T.y1 * A.C.Wc;
            const double w00 = __ldg(Wb + r0 + T.x0), w01 = __ldg(Wb + r0 + T.x1), w10 = __ldg(Wb + r1 + T.x0),
                         w11 = __ldg(Wb + r1 + T.x1);
            const double dx = T.dx, dy = T.dy, ox = 1.0 - dx, oy = 1.0 - dy;
            const float wmf = __fmul_rn(e.p, e.w);
            if (wmf != 0.0f) {   // splat_taps drops a zero weight: no term, as in motion_obj_event_kernel
                const double wm = wmf;
                double sx, sy;
                tap_slopes(ox, oy, dx, dy, w00, w01, w10, w11, sx, sy);
#pragma unroll
                for (int k = 0; k < K; ++k) u[k] += wm * ((double)jx[k] * sx + (double)jy[k] * sy);
            }
            gw = (double)e.p * (oy * (ox * w00 + dx * w01) + dy * (ox * w10 + dx * w11) + c0);
        }
        if (A.grad_w) A.grad_w[i * M + m] = (float)gw;
    });
    cta_add<K, kFlowObjThreads>(u, A.grad + z * K);
}

template <int WARP>
__global__ void __launch_bounds__(kFlowObjThreads) motion_seg_assign_kernel(const ModelArgs A)
{
    __shared__ ModelOf<WARP> mod[kMaxSegModels];
    const int b = blockIdx.y, M = A.M;
    load_models<WARP>(A.params, (int64_t)b * M, M, A.cx, A.cy, mod);
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int Wc = A.C.Wc;
    const int64_t npix = (int64_t)A.C.Hc * Wc;
    const float *Gs = A.G + (int64_t)b * M * npix;
    unsigned oob = 0;
    for_each_event(first, last, [&](int64_t q) { return load_xyt(A.E, q); }, [&](int64_t i, const EvXYT &e) {
        double c[kMaxSegModels], s = 0.0;
#pragma unroll
        for (int m = 0; m < kMaxSegModels; ++m) {
            c[m] = 0.0;
            if (m >= M) continue;
            Taps T;
            float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
            if (model_taps<WARP, false>(A.C, model_event<WARP>(e.x, e.y, e.t, 1.0f), mod[m], oob, T, jx, jy)) {
                const float *G = Gs + m * npix;
                const int64_t r0 = (int64_t)T.y0 * Wc, r1 = (int64_t)T.y1 * Wc;
                const double v = (double)T.ti.x * __ldg(G + r0 + T.x0) + (double)T.ti.y * __ldg(G + r0 + T.x1) +
                                 (double)T.ti.z * __ldg(G + r1 + T.x0) + (double)T.ti.w * __ldg(G + r1 + T.x1);
                c[m] = v < 0.0 ? 0.0 : v;   // a NaN stays NaN
            }
            s += c[m];
        }
        const double den = s + M * A.eps;
        float *row = A.w_out + i * M;
#pragma unroll
        for (int m = 0; m < kMaxSegModels; ++m)
            if (m < M) row[m] = den == 0.0 ? 1.0f / (float)M : (float)((c[m] + A.eps) / den);
    });
}

// shared argument checks and set-up of the segmentation entries: M models per sample, J candidates per model (0: the
// differentiable entries, batch M canvases with the backward's images; else batch M J forward-only canvases)
// The limits of the segmentation entries, which their workspace queries share: 1 <= n_models <= kMaxSegModels and the
// batch_limits of batch M canvases (n_cand 0), or of batch samples with M n_cand candidates each.
static bool seg_limits(int batch, int n_models, int n_cand, int H, int W)
{
    if (n_models < 1 || n_models > kMaxSegModels || batch < 0) return false;
    if (!n_cand) return (int64_t)batch * n_models <= 65535 && batch_limits(batch * n_models, 0, H, W, 1);
    return n_cand >= 1 && (int64_t)n_models * n_cand <= kMaxCandidates && batch_limits(batch, n_models * n_cand, H, W, 1);
}

static int motion_seg_setup(const char *who, const float *x, const float *y, const float *t, const float *p, const float *weights,
                            int n_models, const int64_t *offsets, int batch, int64_t n, int warp, const double *params, int K,
                            double cx, double cy, int H, int W, double sigma, int objective, void *workspace,
                            size_t workspace_bytes, ModelArgs &A, BatchObjWorkspace &ws, BlurTaps &taps, int n_cand = 0)
{
    if (!seg_limits(batch, n_models, n_cand, H, W)) {
        set_error("%s: bad arguments (1 <= n_models <= %d, H, W >= 2, (H+1)(W+1) <= 2^30; batch * n_models <= 65535 canvases; "
                  "candidates: 1 <= n_cand, n_models * n_cand <= %d, batch * n_models * n_cand <= 65535)", who, kMaxSegModels,
                  kMaxCandidates);
        return EVK_E_ARG;
    }
    if (n > 0 && !weights) { set_error("%s: null weights", who); return EVK_E_ARG; }
    const int rc = model_setup(who, x, y, t, nullptr, p, nullptr, false, offsets, n_cand ? batch : batch * n_models, n, warp, params, K,
                               cx, cy, H, W, sigma, objective, 1, (size_t)(H + 1) * (W + 1), n_models * n_cand, workspace,
                               workspace_bytes, A, ws, taps);
    if (rc) return rc;
    A.weights = weights;
    A.M = n_models;
    A.J = n_cand ? n_cand : 1;
    A.wvec4 = n_models % 4 == 0 && ((uintptr_t)weights & 15) == 0;
    return EVK_OK;
}

// ---- dense-flow average-timestamp (Zhu) loss over a batch of samples (evk_flow_timestamp_objective_f32 / _grad_f32) --
// Sample b = events [offsets[b], offsets[b+1]) (clipped to [0, n)) warped by flow[b] with the flow objective's warp and keep
// rule (flow_obj_warp), then the average-timestamp images of events_to_timestamp_image_torch (image.py:286-353) on the
// (H+1)x(W+1) canvas, one per polarity s (p > 0 / p <= 0, a NaN p in neither): S_s = sum tau k, C_s = 1 + sum k over the
// bilinear taps k, T_s = S_s / C_s, and f_b = sum G(T_+)^2 + sum G(T_-)^2.  The 2B images are numbered z = 2b + s, so the
// batched blur, the statistics and the adjoint blur of the other batched losses run over them as over 2B samples.
//   forward:  two v4 reductions per kept event into the 32-byte block {S taps, C taps} of its polarity, [B][2][Hc][Wc][8]
//             (evk_tsimg.cu's layout and arithmetic); a fold to T and C; the blur; per image an f64 sum of G^2.
//   backward: U_s = G(2 g_b G_s) (f64 adjoint blur); (A_s, B_s) = (U_s / C_s, -U_s T_s / C_s) as f32 pairs
//             [B][2][Hc][Wc][2]; per kept event the four pairs of its polarity give dF/dk = tau A + B per tap, then
//             df/dx', df/dy' through the tap weights as in flow_obj_event, spread by flow_obj_spread.
// The accumulator is flow_ts_acc_blocks' (defined with ts_block_add).

template <bool GRAD>
__device__ __forceinline__ void flow_ts_event(const FlowArgs &A, const float *flow, float *acc, const float2 *ab, const EvXYTUP &e,
                                              bool &nonfinite)
{
    FlowSample s;
    Taps T;
    if (!flow_obj_warp(A, flow, e.x, e.y, e.t, 1.0f, s, T, nonfinite)) return;
    const int pol = ts_polarity(e.p);
    if (pol < 0) return;
    const int Wc = A.C.Wc;
    const int64_t plane = (int64_t)A.C.Hc * Wc;
    if (!GRAD) {
        ts_block_add(acc, plane, Wc, pol, T, e.tau);
        return;
    }
    if (pol) ab += plane;
    const float dx = T.dx, dy = T.dy;
    const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
    const int r0 = T.y0 * Wc, r1 = T.y1 * Wc;
    const float2 a00 = __ldg(ab + r0 + T.x0), a01 = __ldg(ab + r0 + T.x1), a10 = __ldg(ab + r1 + T.x0), a11 = __ldg(ab + r1 + T.x1);
    const float tau = e.tau;
    const float q00 = tau * a00.x + a00.y, q01 = tau * a01.x + a01.y, q10 = tau * a10.x + a10.y, q11 = tau * a11.x + a11.y;
    float sx, sy;
    tap_slopes(ox, oy, dx, dy, q00, q01, q10, q11, sx, sy);
    flow_obj_spread(A, acc, s, sx * e.t, sy * e.t);
}

template <bool GRAD>
__global__ void __launch_bounds__(kFlowObjThreads) flow_ts_event_kernel(const FlowArgs A)
{
    const int b = blockIdx.y;
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int64_t npix = (int64_t)A.C.Hc * A.C.Wc;
    const float *flow = A.flow + (int64_t)b * 2 * A.H * A.W;
    float *acc = A.acc + (GRAD ? (int64_t)b * 2 * A.H * A.W * 4 : (int64_t)b * 2 * npix * 8);
    const float2 *ab = GRAD ? A.ab + (int64_t)b * 2 * npix : nullptr;
    bool nonfinite = false;
    for_each_event(first, last, [&](int64_t i) { return load_xytup(A.E, i); },
                   [&](int64_t, const EvXYTUP &e) { flow_ts_event<GRAD>(A, flow, acc, ab, e, nonfinite); });
    if (!GRAD && nonfinite) A.nonfinite[b] = 1u;
}

// blocks -> T and C of every image z = 2b + s (blockIdx.z), tsimg_fold_kernel's arithmetic (the count starts at one, so its
// zero guard never fires); both all-NaN for a sample flagged in nonfinite, so that its f and its gradient are NaN
__global__ void __launch_bounds__(256) flow_ts_fold_kernel(const float *__restrict__ acc, const unsigned *__restrict__ nonfinite,
                                                           int Hc, int Wc, float *__restrict__ ts, float *__restrict__ cnt)
{
    const int64_t npix = (int64_t)Hc * Wc;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    const int64_t k = blockIdx.z * npix + i;
    const float *b = acc + k * 8;
    const int y = i / Wc, x = i - y * Wc;
    float tsum = b[0], csum = b[4];
    if (x > 0) { tsum += b[-8 + 1]; csum += b[-8 + 5]; }
    if (y > 0) { tsum += b[-8 * (int64_t)Wc + 2]; csum += b[-8 * (int64_t)Wc + 6]; }
    if (x > 0 && y > 0) { tsum += b[-8 * ((int64_t)Wc + 1) + 3]; csum += b[-8 * ((int64_t)Wc + 1) + 7]; }
    const float c = __fadd_rn(1.0f, csum);
    const bool bad = nonfinite[blockIdx.z >> 1] != 0;
    ts[k] = bad ? __int_as_float(0x7fc00000) : __fdiv_rn(tsum, c);
    cnt[k] = bad ? __int_as_float(0x7fc00000) : c;
}

// f_b = sum G_+^2 + sum G_-^2 from the f64 sums of cmax_model_stats_kernel (gsums[z][5])
__global__ void flow_ts_final_kernel(const double *gsums, int batch, double *f_out)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) f_out[b] = gsums[8 * (2 * b) + 5] + gsums[8 * (2 * b + 1) + 5];
}

// the coefficient image 2 g_b G_s of df/dG, before the adjoint blur turns it into U_s
__global__ void __launch_bounds__(256) flow_ts_coef_kernel(const float *__restrict__ G, int npix, const float *__restrict__ grad_f,
                                                           double *__restrict__ w)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    const size_t k = (size_t)blockIdx.z * npix + i;
    w[k] = 2.0 * (double)grad_f[blockIdx.z >> 1] * (double)G[k];
}

// dF/dS = U / C and dF/dC = -U T / C per pixel: the pair (A, B) the event pass gathers
__global__ void __launch_bounds__(256) flow_ts_ab_kernel(const float *__restrict__ U, const float *__restrict__ ts,
                                                         const float *__restrict__ cnt, int npix, float2 *__restrict__ ab)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    const size_t k = (size_t)blockIdx.z * npix + i;
    const double u = (double)U[k], c = (double)cnt[k];
    ab[k] = make_float2((float)(u / c), (float)(-u * (double)ts[k] / c));
}

// forward image-space half of the timestamp losses, after their event pass: the 32-byte blocks in ws.acc -> T and C of
// the 2B images (NaN for a sample flagged in ws.nonfinite), the blur, per image an f64 sum of G^2, and f_b
static void ts_obj_forward_tail(const BatchObjWorkspace &ws, int Hc, int Wc, const BlurTaps &taps, int batch, float *ts_out,
                                float *cnt_out, double *f_out, cudaStream_t st)
{
    const int npix = Hc * Wc, images = 2 * batch;
    const dim3 g((npix + 255) / 256, 1, images);
    prof_count(1);
    flow_ts_fold_kernel<<<g, 256, 0, st>>>(ws.acc, ws.nonfinite, Hc, Wc, ts_out, cnt_out);
    batch_obj_blur(ws, ts_out, Hc, Wc, taps, images, st);
    prof_count(2);
    cmax_model_stats_kernel<<<g, 256, 0, st>>>(ws.G, ts_out, npix, OBJ_SOS, 0.0, ws.gsums, ws.gmax, nullptr, nullptr);
    flow_ts_final_kernel<<<(batch + 127) / 128, 128, 0, st>>>(ws.gsums, batch, f_out);
}

// backward image-space half of the timestamp losses, before their event pass: U = G(2 g_b G_s) from the saved T (G
// recomputed, the coefficient image, its adjoint blur into ws.Wimg), then the (A, B) pairs, which go to ws.wt (8 bytes per
// pixel), which the blur has finished reading.  Returns the pairs.
static const float2 *ts_obj_backward_ab(const BatchObjWorkspace &ws, const float *ts_img, const float *cnt_img, int Hc, int Wc,
                                        const BlurTaps &taps, int batch, const float *grad_f, cudaStream_t st)
{
    const int npix = Hc * Wc, images = 2 * batch;
    batch_obj_blur(ws, ts_img, Hc, Wc, taps, images, st);
    const int do_blur = taps.r > 0 || taps.w[0] != 0.0;
    const dim3 g((npix + 255) / 256, 1, images);
    prof_count(do_blur ? 4 : 3);
    flow_ts_coef_kernel<<<g, 256, 0, st>>>(ws.G, npix, grad_f, ws.w);
    if (do_blur) cmax_blur_d_axis0_kernel<<<g, 256, 0, st>>>(ws.w, ws.wt, Hc, Wc, taps);
    cmax_blur_d_axis1_store_kernel<<<g, 256, 0, st>>>(ws.wt, ws.w, Hc, Wc, taps, do_blur, ws.Wimg);
    float2 *ab = reinterpret_cast<float2 *>(ws.wt);
    flow_ts_ab_kernel<<<g, 256, 0, st>>>(ws.Wimg, ts_img, cnt_img, npix, ab);
    return ab;
}

// ---- parametric average-timestamp (Zhu) loss over a batch of samples (evk_motion_timestamp_objective_f32 / _grad_f32) --
// Sample b = events [offsets[b], offsets[b+1]) (clipped to [0, n)) warped by its own model params[b] through model_taps
// (linvel, rotation, xyztheta, affine, homography or camera rotation, f32, as the motion contrast loss warps), with weight 1: an event contributes iff its splat
// there is not zero (finite, 0 < x' < W, 0 < y' < H).  Then the images and f_b of the dense-flow timestamp loss above, on
// the same 2B images z = 2b + s and through the same image-space halves (ts_obj_forward_tail, ts_obj_backward_ab):
//   forward:  two v4 reductions per contributing event into the 32-byte block {S taps, C taps} of its polarity (the
//             arithmetic of flow_ts_event); a non-finite x' or y' contributes nothing, so no sample is ever flagged.
//   backward: per contributing event the four (A, B) pairs of its polarity (L2 gathers), q = tau A + B per tap,
//             df/dx', df/dy' through the tap weights, contracted with the Jacobian rows of model_taps<..., true> and summed
//             in f64 per thread; a CTA reduction and one f64 atomic per component and CTA into grad [B][K], as in
//             motion_obj_event_kernel.
template <int WARP, bool GRAD>
__global__ void __launch_bounds__(kFlowObjThreads) motion_ts_event_kernel(const ModelArgs A)
{
    constexpr int K = model_dims(WARP);
    const int b = blockIdx.y;
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int Wc = A.C.Wc;
    const int64_t npix = (int64_t)A.C.Hc * Wc;
    ModelOf<WARP> M;
    load_model<WARP>(A.params, b, A.cx, A.cy, M);
    float *acc = GRAD ? nullptr : A.acc + b * 2 * npix * 8;
    const float2 *ab = GRAD ? A.ab + b * 2 * npix : nullptr;
    double u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = 0.0;
    unsigned oob = 0;   // a contributing event lies inside the canvas; a non-finite one contributes nothing
    auto load = [&](int64_t i) { return with_depth<WARP>(A.E, i, load_xytup(A.E, i)); };
    for_each_event(first, last, load, [&](int64_t, const Depthed<EvXYTUP, has_depth(WARP)> &e) {
        const int pol = ts_polarity(e.p);
        if (pol < 0) return;
        Taps T;
        float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
        if (!model_taps<WARP, GRAD>(A.C, model_event<WARP>(e.x, e.y, e.t, 1.0f, depth_of(e)), M, oob, T, jx, jy)) return;
        if (!GRAD) {
            ts_block_add(acc, npix, Wc, pol, T, e.tau);
            return;
        }
        const float dx = T.dx, dy = T.dy;
        const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
        const float2 *abs_ = pol ? ab + npix : ab;
        const int64_t r0 = (int64_t)T.y0 * Wc, r1 = (int64_t)T.y1 * Wc;
        const float2 a00 = __ldg(abs_ + r0 + T.x0), a01 = __ldg(abs_ + r0 + T.x1), a10 = __ldg(abs_ + r1 + T.x0),
                     a11 = __ldg(abs_ + r1 + T.x1);
        const double tau = e.tau;
        const double q00 = tau * a00.x + a00.y, q01 = tau * a01.x + a01.y, q10 = tau * a10.x + a10.y, q11 = tau * a11.x + a11.y;
        double sx, sy;
        tap_slopes<double>(ox, oy, dx, dy, q00, q01, q10, q11, sx, sy);
#pragma unroll
        for (int k = 0; k < K; ++k) u[k] += (double)jx[k] * sx + (double)jy[k] * sy;
    });
    if (GRAD) cta_add<K, kFlowObjThreads>(u, A.grad + (int64_t)b * K);
}

// the candidates entry's workspace for `images` = 2 batch n_cand images: the forward-only carve (no f64 adjoint images;
// the T images go to its Wimg), then the C images the fold writes, which nothing reads
static size_t motion_ts_cand_head(int images, int H, int W)
{
    return batch_obj_carve(nullptr, images, H, W, flow_ts_acc_blocks(H, W), nullptr, false);
}
static size_t motion_ts_cand_bytes(int images, int H, int W)
{
    return motion_ts_cand_head(images, H, W) + align_up((size_t)images * (H + 1) * (W + 1) * sizeof(float), 256);
}

// ---- many parameter vectors per sample in one event pass (evk_motion_timestamp_candidates_f32) --------------------
// The grid search and the line search of a batched fit of the timestamp loss score n_cand parameter vectors of every
// sample.  On the (slices, batch) grid, each CTA takes its sample's n_cand x K candidates into shared memory, reads each
// event ONCE (x, y, t, tau, p: 20 B) and, under every candidate that keeps it, makes the two v4 reductions of
// motion_ts_event_kernel's forward into the 32-byte {S, C} block of its polarity, image pair z = 2 (b n_cand + j) + s of
// [batch][n_cand][2][Hc][Wc][8].  ts_obj_forward_tail then treats the batch x n_cand pairs as the samples of
// evk_motion_timestamp_objective_f32, so f comes out in [batch][n_cand] order.
template <int WARP>
struct TsCandEvent {
    Event<WARP> e;   // splat weight 1
    float tau;
    int pol = -1;    // ts_polarity; -1 also past the end of the sample
};

template <int WARP>
__global__ void __launch_bounds__(kFlowObjThreads) motion_ts_cand_kernel(const ModelArgs A)
{
    __shared__ ModelOf<WARP> cand[kMaxCandidates];
    const int b = blockIdx.y, J = A.J;
    load_models<WARP>(A.params, (int64_t)b * J, J, A.cx, A.cy, cand);
    int64_t first, last;
    sample_range(A.E, b, first, last);
    const int Wc = A.C.Wc;
    const int64_t npix = (int64_t)A.C.Hc * Wc;
    float *acc = A.acc + (int64_t)b * J * 2 * npix * 8;
    unsigned oob = 0;   // as in motion_ts_event_kernel: a contributing event lies inside the canvas
    auto load = [&](int64_t q) {
        const auto r = with_depth<WARP>(A.E, q, load_xytup(A.E, q));
        TsCandEvent<WARP> c;
        c.e = model_event<WARP>(r.x, r.y, r.t, 1.0f, depth_of(r));
        c.tau = r.tau;
        c.pol = ts_polarity(r.p);
        return c;
    };
    for_each_event_batch(first, last, load, [&](const TsCandEvent<WARP> (&e)[kBatch], int) {
        for (int j = 0; j < J; ++j) {
            const ModelOf<WARP> M = cand[j];
            float *accj = acc + (int64_t)j * 2 * npix * 8;
#pragma unroll
            for (int k = 0; k < kBatch; ++k) {
                Taps T;
                float jx[jac_dims(WARP)], jy[jac_dims(WARP)];
                if (e[k].pol < 0 || !model_taps<WARP, false>(A.C, e[k].e, M, oob, T, jx, jy)) continue;
                ts_block_add(accj, npix, Wc, e[k].pol, T, e[k].tau);
            }
        }
    });
}

}  // namespace evk

extern "C" {

size_t evk_cmax_workspace_bytes(int Hs, int Ws)
{
    if (Hs < 1 || Ws < 1) return 0;
    return evk::carve(nullptr, Hs, Ws, nullptr);
}

static int linvel_objective_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                  double p_scale, double vx, double vy, double t_ref, int Hm, int Wm, int Hs, int Ws,
                                  double sigma, unsigned flags, int objective, double obj_param, double *result,
                                  float *iwe_out, float *diwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_linvel_objective_f64", sigma)) return rc;
    if (n > 0 && (!x || !y || !t || !p)) { set_error("evk_cmax_linvel_objective_f64: null event array"); return EVK_E_ARG; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.vx = vx; A.vy = vy; A.t_ref = t_ref; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    return run_cmax<WARP_LINVEL_F64>(A, sigma, flags, objective, obj_param, result, iwe_out, diwe_out, workspace,
                                     workspace_bytes, static_cast<cudaStream_t>(stream));
}

static int linvel_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n,
                                  float p_scale, float vx, float vy, int Hm, int Wm, int Hs, int Ws, double sigma,
                                  unsigned flags, int objective, double obj_param, double *result, float *iwe_out,
                                  float *diwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_linvel_objective_f32", sigma)) return rc;
    if (n > 0 && (!x || !y || !t_rel || !p)) { set_error("evk_cmax_linvel_objective_f32: null event array"); return EVK_E_ARG; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t_rel; A.p = p; A.n = n;
    A.vx = vx; A.vy = vy; A.t_ref = 0.0; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    return run_cmax<WARP_LINVEL_F32>(A, sigma, flags, objective, obj_param, result, iwe_out, diwe_out, workspace,
                                     workspace_bytes, static_cast<cudaStream_t>(stream));
}

// The objective entries' result has 12 slots, the variance entries' 8; the variance tails fill the first 8, so the objective
// entries zero [8..11] for EVK_OBJ_VARIANCE (n results of `stride` doubles)
static int zero_variance_stats(int rc, int objective, double *result, int n, int stride, void *stream)
{
    using namespace evk;
    if (rc || objective != OBJ_VARIANCE || !result) return rc;
    EVK_CUDA(cudaMemset2DAsync(result + 8, (size_t)stride * sizeof(double), 0, 4 * sizeof(double), n,
                               static_cast<cudaStream_t>(stream)));
    return EVK_OK;
}

int evk_cmax_linvel_objective_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                  double p_scale, double vx, double vy, double t_ref, int Hm, int Wm, int Hs, int Ws,
                                  double sigma, unsigned flags, int objective, double obj_param, double *result,
                                  float *iwe_out, float *diwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    const int rc = linvel_objective_f64(x, y, t, p, n, p_scale, vx, vy, t_ref, Hm, Wm, Hs, Ws, sigma, flags, objective, obj_param,
                                        result, iwe_out, diwe_out, workspace, workspace_bytes, stream);
    return zero_variance_stats(rc, objective, result, 1, 12, stream);
}

int evk_cmax_linvel_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n,
                                  float p_scale, float vx, float vy, int Hm, int Wm, int Hs, int Ws, double sigma,
                                  unsigned flags, int objective, double obj_param, double *result, float *iwe_out,
                                  float *diwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    const int rc = linvel_objective_f32(x, y, t_rel, p, n, p_scale, vx, vy, Hm, Wm, Hs, Ws, sigma, flags, objective, obj_param,
                                        result, iwe_out, diwe_out, workspace, workspace_bytes, stream);
    return zero_variance_stats(rc, objective, result, 1, 12, stream);
}

int evk_cmax_linvel_variance_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                 double p_scale, double vx, double vy, double t_ref, int Hm, int Wm, int Hs, int Ws,
                                 double sigma, unsigned flags, double *result, float *iwe_out, float *diwe_out,
                                 void *workspace, size_t workspace_bytes, void *stream)
{
    return linvel_objective_f64(x, y, t, p, n, p_scale, vx, vy, t_ref, Hm, Wm, Hs, Ws, sigma, flags, 0, 0.0, result,
                                         iwe_out, diwe_out, workspace, workspace_bytes, stream);
}

int evk_cmax_linvel_variance_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n,
                                 float p_scale, float vx, float vy, int Hm, int Wm, int Hs, int Ws, double sigma,
                                 unsigned flags, double *result, float *iwe_out, float *diwe_out, void *workspace,
                                 size_t workspace_bytes, void *stream)
{
    return linvel_objective_f32(x, y, t_rel, p, n, p_scale, vx, vy, Hm, Wm, Hs, Ws, sigma, flags, 0, 0.0, result,
                                         iwe_out, diwe_out, workspace, workspace_bytes, stream);
}

int evk_cmax_linvel_partial_f64(const double *x, const double *y, const double *t, const double *p, int64_t n, double p_scale,
                                double vx, double vy, double t_ref, int Hm, int Wm, int Hs, int Ws, unsigned flags,
                                float *images_out, unsigned long long *oob_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (!images_out || (n > 0 && (!x || !y || !t || !p))) { set_error("evk_cmax_linvel_partial_f64: null array"); return EVK_E_ARG; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.vx = vx; A.vy = vy; A.t_ref = t_ref; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    return run_cmax<WARP_LINVEL_F64>(A, 0.0, flags, 0, 0.0, nullptr, nullptr, nullptr, workspace, workspace_bytes,
                                     static_cast<cudaStream_t>(stream), images_out, oob_out);
}

int evk_cmax_linvel_partial_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n, float p_scale,
                                float vx, float vy, int Hm, int Wm, int Hs, int Ws, unsigned flags, float *images_out,
                                unsigned long long *oob_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (!images_out || (n > 0 && (!x || !y || !t_rel || !p))) { set_error("evk_cmax_linvel_partial_f32: null array"); return EVK_E_ARG; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t_rel; A.p = p; A.n = n;
    A.vx = vx; A.vy = vy; A.t_ref = 0.0; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    return run_cmax<WARP_LINVEL_F32>(A, 0.0, flags, 0, 0.0, nullptr, nullptr, nullptr, workspace, workspace_bytes,
                                     static_cast<cudaStream_t>(stream), images_out, oob_out);
}

int evk_cmax_peer_tail_f32(const float *const *peer_images, const unsigned long long *const *peer_oob, int world, int Hc, int Wc,
                           double sigma, unsigned flags, double *result, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_peer_tail_f32", sigma)) return rc;
    if (!peer_images || !peer_oob || world < 1 || world > kMaxCmaxPeers || Hc < 2 || Wc < 2 || !result || !workspace) {
        set_error("evk_cmax_peer_tail_f32: bad arguments (1 <= world <= %d)", kMaxCmaxPeers);
        return EVK_E_ARG;
    }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_cmax_peer_tail_f32: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hc - 1, Wc - 1, &ws);
    if (workspace_bytes < need) { set_error("evk_cmax_peer_tail_f32: workspace of %zu bytes required", need); return EVK_E_WORKSPACE; }
    BlurTaps taps{};
    double mix_a = 1.0, mix_b = 0.0;
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
        if (taps.r > kFusedMaxR) { set_error("evk_cmax_peer_tail_f32: blur radius %d > %d", taps.r, kFusedMaxR); return EVK_E_UNSUPPORTED; }
        if (!(flags & EVK_CMAX_NO_CHANNEL_MIX)) mix_coeffs(taps, &mix_a, &mix_b);
    }
    CmaxPeers P{};
    P.world = world;
    for (int r = 0; r < world; ++r) {
        if (!peer_images[r] || !peer_oob[r]) { set_error("evk_cmax_peer_tail_f32: peer %d: null pointer", r); return EVK_E_ARG; }
        P.img[r] = peer_images[r];
        P.oob[r] = peer_oob[r];
    }
    // the sums and the ticket of the tail (gsums .. oob are contiguous)
    EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)((char *)(ws.oob + 1) - (char *)ws.gsums), st));
    prof_count(1);
    dim3 tgrid((Wc + kTileX - 1) / kTileX, (Hc + kTileY - 1) / kTileY), tblock(kTileX, kTileY);
    cmax_fused_var_tail_kernel_t<true><<<tgrid, tblock, 0, st>>>(P, nullptr, nullptr, 1, Hc, Wc, taps, do_blur, (flags & EVK_CMAX_WANT_GRAD) ? 1 : 0,
                                                                  mix_a, mix_b, nullptr, nullptr, ws.sums, ws.gmax, ws.oob, result, ws.w);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_flow_variance_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                               const float *flow, float t0, int Hs, int Ws, double sigma, unsigned flags,
                               double *result, float *iwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_flow_variance_f32", sigma)) return rc;
    if (!flow || (n > 0 && (!x || !y || !t || !p))) { set_error("evk_cmax_flow_variance_f32: null array"); return EVK_E_ARG; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.flow = flow; A.flow_t0 = t0; A.p_scale = 1.0;
    A.Hm = Hs; A.Wm = Ws; A.Hc = Hs + 1; A.Wc = Ws + 1;
    return run_cmax<WARP_FLOW_F32>(A, sigma, flags, 0, 0.0, result, iwe_out, nullptr, workspace, workspace_bytes,
                                   static_cast<cudaStream_t>(stream));
}

static int iwe_objective(const float *iwe, const float *diwe, int Hc, int Wc, double sigma, unsigned flags, int objective,
                         double obj_param, double *result, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_iwe_objective_f32", sigma)) return rc;
    if (!iwe || !result || !workspace || Hc < 2 || Wc < 2) { set_error("evk_iwe_objective_f32: bad arguments"); return EVK_E_ARG; }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_iwe_objective_f32: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hc - 1, Wc - 1, &ws);
    if (workspace_bytes < need) { set_error("evk_iwe_objective_f32: workspace of %zu bytes required", need); return EVK_E_WORKSPACE; }
    const int npix = Hc * Wc;
    const bool grad = (flags & EVK_CMAX_WANT_GRAD) != 0 && diwe != nullptr;
    EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)((char *)(ws.oob + 1) - (char *)ws.gsums), st));
    prof_count(1);
    cmax_planar_kernel<<<(npix + 255) / 256, 256, 0, st>>>(iwe, grad ? diwe : nullptr, npix, ws.I, ws.D0, ws.D1, ws.sums);
    return launch_tail(ws, Hc, Wc, sigma, flags, objective, obj_param, grad, result, st);
}

int evk_iwe_objective_f32(const float *iwe, const float *diwe, int Hc, int Wc, double sigma, unsigned flags, int objective,
                          double obj_param, double *result, void *workspace, size_t workspace_bytes, void *stream)
{
    const int rc = iwe_objective(iwe, diwe, Hc, Wc, sigma, flags, objective, obj_param, result, workspace, workspace_bytes, stream);
    return zero_variance_stats(rc, objective, result, 1, 12, stream);
}

int evk_variance_objective_f32(const float *iwe, const float *diwe, int Hc, int Wc, double sigma, unsigned flags,
                               double *result, void *workspace, size_t workspace_bytes, void *stream)
{
    return iwe_objective(iwe, diwe, Hc, Wc, sigma, flags, 0, 0.0, result, workspace, workspace_bytes, stream);
}

int evk_gaussian_blur_f32(const float *img, int H, int W, double sigma, float *out, float *tmp, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_gaussian_blur_f32", sigma)) return rc;
    if (!img || !out || !tmp || H < 1 || W < 1) { set_error("evk_gaussian_blur_f32: bad arguments"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    BlurTaps taps{};
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
    }
    const int g = (H * W + 255) / 256;
    prof_count(do_blur ? 2 : 1);
    if (do_blur) cmax_blur_axis0_kernel<<<g, 256, 0, st>>>(img, tmp, H, W, taps);
    cmax_blur_axis1_store_kernel<<<g, 256, 0, st>>>(tmp, img, H, W, taps, do_blur, out);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_linvel_objective_batch_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                        double p_scale, const double *params_host, int n_params, double t_ref, int Hm, int Wm,
                                        int Hs, int Ws, double sigma, unsigned flags, int objective, double obj_param,
                                        double *results, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_linvel_objective_batch_f64", sigma)) return rc;
    if (n < 0 || (n > 0 && (!x || !y || !t || !p)) || !params_host || n_params < 1 || n_params > kMaxCandidates || !results || !workspace) {
        set_error("evk_cmax_linvel_objective_batch_f64: bad arguments (1 <= n_params <= %d)", kMaxCandidates);
        return EVK_E_ARG;
    }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_cmax batch: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hs, Ws, &ws);
    if (workspace_bytes < need) { set_error("evk_cmax batch: workspace of %zu bytes required", need); return EVK_E_WORKSPACE; }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t_ref = t_ref; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    A.abs_polarity = (flags & EVK_CMAX_ABS_POLARITY) ? 1 : 0;
    A.replicas = 1; A.acc = ws.acc; A.oob = ws.oob;
    const int npix = A.Hc * A.Wc;
    const bool grad = (flags & EVK_CMAX_WANT_GRAD) != 0;
    Candidates C{};
    C.n = n_params;
    for (int k = 0; k < n_params; ++k) { C.vx[k] = params_host[2 * k]; C.vy[k] = params_host[2 * k + 1]; }
    // bsums, btickets, gsums, gmax, sums, oob and the accumulators are contiguous: one memset
    EVK_CUDA(cudaMemsetAsync(ws.bsums, 0, (size_t)((char *)ws.acc - (char *)ws.bsums) + (size_t)n_params * npix * kBlockFloats * sizeof(float), st));
    if (n > 0) {
        ProfScope prof(st);
        prof_count(1);
        if (grad) cmax_scatter_batch_kernel<WARP_LINVEL_F64, true><<<grid_for(cmax_scatter_batch_kernel<WARP_LINVEL_F64, true>, 256, n, 256 * 2), 256, 0, st>>>(A, C);
        else cmax_scatter_batch_kernel<WARP_LINVEL_F64, false><<<grid_for(cmax_scatter_batch_kernel<WARP_LINVEL_F64, false>, 256, n, 256 * 2), 256, 0, st>>>(A, C);
        EVK_CUDA(cudaGetLastError());
    }
    BlurTaps taps{};
    double mix_a = 1.0, mix_b = 0.0;
    const int do_blur = sigma > 0.0;
    if (do_blur) {
        int rc = make_taps(sigma, &taps);
        if (rc) return rc;
        if (!(flags & EVK_CMAX_NO_CHANNEL_MIX)) mix_coeffs(taps, &mix_a, &mix_b);
    }
    if (objective == OBJ_VARIANCE && taps.r <= kFusedMaxR) {
        // all candidates' tails in ONE launch (blockIdx.z = candidate)
        prof_count(1);
        dim3 tgrid((A.Wc + kTileX - 1) / kTileX, (A.Hc + kTileY - 1) / kTileY, n_params), tblock(kTileX, kTileY);
        cmax_fused_var_tail_kernel_t<false><<<tgrid, tblock, 0, st>>>(CmaxPeers{}, ws.acc, nullptr, 1, A.Hc, A.Wc, taps, do_blur, grad ? 1 : 0, mix_a, mix_b, nullptr,
                                                               nullptr, ws.bsums, ws.btickets, ws.oob, results);
        EVK_CUDA(cudaGetLastError());
        return zero_variance_stats(EVK_OK, objective, results, n_params, 12, stream);
    }
    for (int k = 0; k < n_params; ++k) {
        // per-candidate image-space tail on the shared scratch images (stream-ordered)
        EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)((char *)ws.oob - (char *)ws.gsums), st));   // keep the oob counter
        prof_count(1);
        cmax_gather_kernel<<<(npix + 255) / 256, 256, 0, st>>>(ws.acc + (size_t)k * npix * kBlockFloats, nullptr, 1, A.Hc, A.Wc, ws.I, ws.D0,
                                                                ws.D1, nullptr, nullptr, ws.sums);
        int rc = launch_tail(ws, A.Hc, A.Wc, sigma, flags, objective, obj_param, grad, results + 12 * k, st);
        if (rc) return rc;
    }
    return zero_variance_stats(EVK_OK, objective, results, n_params, 12, stream);
}

int evk_cmax_warp_objective_f64(const double *x, const double *y, const double *t, const double *p, int64_t n, double p_scale,
                                int warp, const double *model, double t_ref, int Hm, int Wm, int Hs, int Ws, double sigma,
                                unsigned flags, int objective, double obj_param, double *result, float *iwe_out,
                                void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_warp_objective_f64", sigma)) return rc;
    if (n > 0 && (!x || !y || !t || !p)) { set_error("evk_cmax_warp_objective_f64: null event array"); return EVK_E_ARG; }
    CmaxArgs A{};
    int rc = read_model(warp, model, &A.model, nullptr);
    if (rc) return rc;
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t_ref = t_ref; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (warp == EVK_WARP_ROTATION)
        return run_model<WARP_ROTATION_F64>(A, sigma, flags, objective, obj_param, result, iwe_out, workspace, workspace_bytes, st);
    return run_model<WARP_XYZTHETA_F64>(A, sigma, flags, objective, obj_param, result, iwe_out, workspace, workspace_bytes, st);
}

int evk_cmax_warp_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, int64_t n, float p_scale,
                                int warp, const double *model, int Hm, int Wm, int Hs, int Ws, double sigma, unsigned flags,
                                int objective, double obj_param, double *result, float *iwe_out, void *workspace,
                                size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_warp_objective_f32", sigma)) return rc;
    if (n > 0 && (!x || !y || !t_rel || !p)) { set_error("evk_cmax_warp_objective_f32: null event array"); return EVK_E_ARG; }
    CmaxArgs A{};
    int rc = read_model(warp, model, &A.model, nullptr);
    if (rc) return rc;
    A.x = x; A.y = y; A.t = t_rel; A.p = p; A.n = n;
    A.t_ref = 0.0; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (warp == EVK_WARP_ROTATION)
        return run_model<WARP_ROTATION_F32>(A, sigma, flags, objective, obj_param, result, iwe_out, workspace, workspace_bytes, st);
    return run_model<WARP_XYZTHETA_F32>(A, sigma, flags, objective, obj_param, result, iwe_out, workspace, workspace_bytes, st);
}

int evk_cmax_warp_objective_batch_f64(const double *x, const double *y, const double *t, const double *p, int64_t n,
                                      double p_scale, int warp, const double *models_host, int n_models, double t_ref, int Hm,
                                      int Wm, int Hs, int Ws, double sigma, unsigned flags, int objective, double obj_param,
                                      double *results, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (int rc = check_sigma("evk_cmax_warp_objective_batch_f64", sigma)) return rc;
    if (n < 0 || (n > 0 && (!x || !y || !t || !p)) || !models_host || n_models < 1 || n_models > kMaxCandidates || !results ||
        !workspace || Hs < 1 || Ws < 1) {
        set_error("evk_cmax_warp_objective_batch_f64: bad arguments (1 <= n_models <= %d)", kMaxCandidates);
        return EVK_E_ARG;
    }
    if (objective < OBJ_VARIANCE || objective > OBJ_SOSA) { set_error("evk_cmax_warp: unknown objective %d", objective); return EVK_E_ARG; }
    if (((uintptr_t)workspace & 255) != 0) { set_error("evk_cmax_warp batch: workspace must be 256-byte aligned"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CmaxWorkspace ws;
    const size_t need = carve(workspace, Hs, Ws, &ws);
    if (workspace_bytes < need) { set_error("evk_cmax_warp batch: workspace of %zu bytes required", need); return EVK_E_WORKSPACE; }
    ModelCandidates C{};
    C.n = n_models;
    int nd = 0;
    for (int k = 0; k < n_models; ++k) {
        int rc = read_model(warp, models_host + (size_t)k * (warp == EVK_WARP_ROTATION ? 3 : 6), &C.m[k], &nd);
        if (rc) return rc;
    }
    CmaxArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t_ref = t_ref; A.p_scale = p_scale;
    A.Hm = Hm; A.Wm = Wm; A.Hc = Hs + 1; A.Wc = Ws + 1;
    A.abs_polarity = (flags & EVK_CMAX_ABS_POLARITY) ? 1 : 0;
    A.replicas = 1; A.acc = ws.acc; A.oob = ws.oob;
    const int npix = A.Hc * A.Wc;
    // bsums, btickets, gsums, gmax, sums, oob and the accumulators are contiguous: one memset
    EVK_CUDA(cudaMemsetAsync(ws.bsums, 0, (size_t)((char *)ws.acc - (char *)ws.bsums) + (size_t)n_models * npix * kBlockFloats * sizeof(float), st));
    if (n > 0) {
        ProfScope prof(st);
        prof_count(1);
        if (warp == EVK_WARP_ROTATION)
            cmax_model_batch_kernel<WARP_ROTATION_F64><<<grid_for(cmax_model_batch_kernel<WARP_ROTATION_F64>, 256, n, 256 * 2), 256, 0, st>>>(A, C);
        else
            cmax_model_batch_kernel<WARP_XYZTHETA_F64><<<grid_for(cmax_model_batch_kernel<WARP_XYZTHETA_F64>, 256, n, 256 * 2), 256, 0, st>>>(A, C);
        EVK_CUDA(cudaGetLastError());
    }
    for (int k = 0; k < n_models; ++k) {
        // per-candidate image-space tail on the shared scratch images (stream-ordered); the oob counter is kept
        EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)((char *)ws.oob - (char *)ws.gsums), st));
        prof_count(1);
        cmax_gather_kernel<<<(npix + 255) / 256, 256, 0, st>>>(ws.acc + (size_t)k * npix * kBlockFloats, nullptr, 1, A.Hc, A.Wc, ws.I, ws.D0,
                                                                ws.D1, nullptr, nullptr, ws.sums);
        int rc = model_tail(ws, A.Hc, A.Wc, sigma, objective, obj_param, nullptr, st);
        if (rc) return rc;
        cmax_model_final_kernel<<<1, 1, 0, st>>>(objective, ws.gsums, ws.gmax, ws.sums, ws.oob, npix, ws.sums + 1, 4, 0, results + 16 * k);
        EVK_CUDA(cudaGetLastError());
    }
    return EVK_OK;
}

size_t evk_cmax_flow_objective_workspace_bytes(int batch, int H, int W)
{
    if (!evk::batch_limits(batch, 0, H, W, 1)) return 0;
    return evk::batch_obj_carve(nullptr, batch, H, W, evk::flow_obj_acc_blocks(H, W), nullptr);
}

int evk_cmax_flow_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                int batch, int64_t n_events, const float *flow, int H, int W, double sigma, int objective,
                                double obj_param, double *f_out, float *iwe_out, void *workspace, size_t workspace_bytes,
                                void *stream)
{
    using namespace evk;
    FlowArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = flow_setup("evk_cmax_flow_objective_f32", x, y, t_rel, nullptr, p, offsets, batch, n_events, flow, H, W, sigma,
                        objective, 1, flow_obj_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !iwe_out)) { set_error("evk_cmax_flow_objective_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc;
    EVK_CUDA(batch_obj_zero(ws, batch, npix, 4, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        flow_obj_event_kernel<false><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
    }
    batch_obj_forward_tail(ws, Hc, Wc, taps, batch, objective, obj_param, iwe_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_flow_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                     int batch, int64_t n_events, const float *flow, int H, int W, double sigma, int objective,
                                     double obj_param, const float *iwe, const float *grad_f, float *grad_flow, void *workspace,
                                     size_t workspace_bytes, void *stream)
{
    using namespace evk;
    FlowArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = flow_setup("evk_cmax_flow_objective_grad_f32", x, y, t_rel, nullptr, p, offsets, batch, n_events, flow, H, W, sigma,
                        objective, 1, flow_obj_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_flow)) { set_error("evk_cmax_flow_objective_grad_f32: null array"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1;
    const int64_t planes = (int64_t)batch * 2;
    EVK_CUDA(cudaMemsetAsync(ws.acc, 0, (size_t)planes * H * W * 4 * sizeof(float), st));
    // W = G(g_b C_b): recompute G from the saved IWE, the coefficient image, its blur
    batch_obj_backward_W(ws, iwe, Hc, Wc, taps, batch, objective, obj_param, grad_f, st);
    A.Wimg = ws.Wimg;
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        flow_obj_event_kernel<true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
    }
    prof_count(1);
    flow_obj_grad_fold_kernel<<<grid_simple(planes * H * W, 256), 256, 0, st>>>(ws.acc, grad_flow, planes, H, W);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_cmax_grid_flow_objective_workspace_bytes(int batch, int gh, int gw, int H, int W)
{
    if (!evk::grid_flow_limits(batch, 0, gh, gw, H, W)) return 0;
    return evk::batch_obj_carve(nullptr, batch, H, W, (size_t)(H + 1) * (W + 1), nullptr);
}

int evk_cmax_grid_flow_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                     int batch, int64_t n_events, const float *grid_flow, int gh, int gw, int H, int W,
                                     double sigma, int objective, double obj_param, double *f_out, float *iwe_out,
                                     void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup("evk_cmax_grid_flow_objective_f32", x, y, t_rel, nullptr, p, offsets, batch, n_events, grid_flow, 0,
                             gh, gw, H, W, sigma, objective, 1, (size_t)(H + 1) * (W + 1), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !iwe_out)) { set_error("evk_cmax_grid_flow_objective_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    return grid_flow_forward(A, ws, taps, batch, objective, obj_param, iwe_out, f_out, static_cast<cudaStream_t>(stream));
}

int evk_cmax_grid_flow_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                          const int64_t *offsets, int batch, int64_t n_events, const float *grid_flow, int gh,
                                          int gw, int H, int W, double sigma, int objective, double obj_param, const float *iwe,
                                          const float *grad_f, float *grad_grid, void *workspace, size_t workspace_bytes,
                                          void *stream)
{
    using namespace evk;
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup("evk_cmax_grid_flow_objective_grad_f32", x, y, t_rel, nullptr, p, offsets, batch, n_events, grid_flow,
                             0, gh, gw, H, W, sigma, objective, 1, (size_t)(H + 1) * (W + 1), workspace, workspace_bytes, A, ws,
                             taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_grid)) {
        set_error("evk_cmax_grid_flow_objective_grad_f32: null array");
        return EVK_E_ARG;
    }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t nodes = (int64_t)batch * 2 * gh * gw;
    // the f64 node sums live in the accumulator, which the backward has no other use for ((H+1)(W+1) 16 B >= 2 gh gw 8 B)
    A.grad = reinterpret_cast<double *>(ws.acc);
    EVK_CUDA(cudaMemsetAsync(A.grad, 0, (size_t)nodes * sizeof(double), st));
    batch_obj_backward_W(ws, iwe, H + 1, W + 1, taps, batch, objective, obj_param, grad_f, st);
    A.F.Wimg = ws.Wimg;
    return grid_flow_node_grad<false>(A, batch, grad_grid, st);
}

size_t evk_cmax_grid_flow_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W)
{
    if (!evk::grid_flow_limits(batch, n_cand < 1 ? -1 : n_cand, gh, gw, H, W)) return 0;
    return evk::batch_obj_carve(nullptr, batch * n_cand, H, W, (size_t)(H + 1) * (W + 1), nullptr, false);
}

int evk_cmax_grid_flow_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                      int batch, int64_t n_events, const float *cand, int n_cand, int gh, int gw, int H, int W,
                                      double blur_sigma, int objective, double obj_param, double *f_out, void *workspace,
                                      size_t workspace_bytes, void *stream)
{
    using namespace evk;
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup("evk_cmax_grid_flow_candidates_f32", x, y, t_rel, nullptr, p, offsets, batch, n_events, cand,
                             n_cand < 1 ? -1 : n_cand, gh, gw, H, W, blur_sigma, objective, 1, (size_t)(H + 1) * (W + 1), workspace,
                             workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && !f_out) { set_error("evk_cmax_grid_flow_candidates_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    // the folded images go to ws.Wimg, which a forward-only workspace has no other use for
    return grid_flow_forward(A, ws, taps, batch, objective, obj_param, ws.Wimg, f_out, static_cast<cudaStream_t>(stream));
}

size_t evk_cmax_depth_grid_objective_workspace_bytes(int batch, int gh, int gw, int H, int W)
{
    return evk_cmax_grid_flow_objective_workspace_bytes(batch, gh, gw, H, W);
}

int evk_cmax_depth_grid_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                      const int64_t *offsets, int batch, int64_t n_events, const double *motion, double cx,
                                      double cy, const float *inv_depth_grid, int gh, int gw, int H, int W, double sigma,
                                      int objective, double obj_param, double *f_out, float *iwe_out, void *workspace,
                                      size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_depth_grid_objective_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, nullptr, p, offsets, batch, n_events, motion, cx, cy, inv_depth_grid, 0, gh, gw, H,
                              W, sigma, objective, 1, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !iwe_out)) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    return depth_grid_forward(D, ws, taps, batch, objective, obj_param, iwe_out, f_out, static_cast<cudaStream_t>(stream));
}

int evk_cmax_depth_grid_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                           const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                           double cx, double cy, const float *inv_depth_grid, int gh, int gw, int H, int W,
                                           double sigma, int objective, double obj_param, const float *iwe,
                                           const float *grad_f, float *grad_grid, void *workspace, size_t workspace_bytes,
                                           void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_depth_grid_objective_grad_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, nullptr, p, offsets, batch, n_events, motion, cx, cy, inv_depth_grid, 0, gh, gw, H,
                              W, sigma, objective, 1, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_grid)) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the f64 node sums live in the accumulator, which the backward has no other use for ((H+1)(W+1) 16 B >= gh gw 8 B)
    D.G.grad = reinterpret_cast<double *>(ws.acc);
    EVK_CUDA(cudaMemsetAsync(D.G.grad, 0, (size_t)batch * gh * gw * sizeof(double), st));
    batch_obj_backward_W(ws, iwe, H + 1, W + 1, taps, batch, objective, obj_param, grad_f, st);
    D.G.F.Wimg = ws.Wimg;
    return depth_grid_node_grad<false>(D, batch, grad_grid, st);
}

size_t evk_cmax_depth_grid_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W)
{
    return evk_cmax_grid_flow_candidates_workspace_bytes(batch, n_cand, gh, gw, H, W);
}

int evk_cmax_depth_grid_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, const double *motion, double cx,
                                       double cy, const float *cand, int n_cand, int gh, int gw, int H, int W,
                                       double blur_sigma, int objective, double obj_param, double *f_out, void *workspace,
                                       size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_depth_grid_candidates_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, nullptr, p, offsets, batch, n_events, motion, cx, cy, cand, n_cand < 1 ? -1 : n_cand,
                              gh, gw, H, W, blur_sigma, objective, 1, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    // the folded images go to ws.Wimg, which a forward-only workspace has no other use for
    return depth_grid_forward(D, ws, taps, batch, objective, obj_param, ws.Wimg, f_out, static_cast<cudaStream_t>(stream));
}

size_t evk_cmax_depth_grid_joint_grad_workspace_bytes(int batch, int gh, int gw, int H, int W)
{
    return evk_cmax_depth_grid_objective_workspace_bytes(batch, gh, gw, H, W);
}

int evk_cmax_depth_grid_joint_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, const double *motion, double cx,
                                       double cy, const float *inv_depth_grid, int gh, int gw, int H, int W, double sigma,
                                       int objective, double obj_param, const float *iwe, const float *grad_f,
                                       float *grad_grid, double *grad_motion, void *workspace, size_t workspace_bytes,
                                       void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_depth_grid_joint_grad_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, nullptr, p, offsets, batch, n_events, motion, cx, cy, inv_depth_grid, 0, gh, gw, H,
                              W, sigma, objective, 1, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_grid || !grad_motion)) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the node sums in the accumulator, as in evk_cmax_depth_grid_objective_grad_f32
    D.G.grad = reinterpret_cast<double *>(ws.acc);
    D.grad_motion = grad_motion;
    EVK_CUDA(cudaMemsetAsync(D.G.grad, 0, (size_t)batch * gh * gw * sizeof(double), st));
    EVK_CUDA(cudaMemsetAsync(grad_motion, 0, (size_t)batch * 6 * sizeof(double), st));
    batch_obj_backward_W(ws, iwe, H + 1, W + 1, taps, batch, objective, obj_param, grad_f, st);
    D.G.F.Wimg = ws.Wimg;
    return depth_grid_node_grad<false, true>(D, batch, grad_grid, st);
}

size_t evk_cmax_depth_grid_joint_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W)
{
    return evk_cmax_depth_grid_candidates_workspace_bytes(batch, n_cand, gh, gw, H, W);
}

int evk_cmax_depth_grid_joint_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                             const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                             double cx, double cy, const float *cand, int n_cand, int gh, int gw, int H, int W,
                                             double blur_sigma, int objective, double obj_param, double *f_out, void *workspace,
                                             size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_depth_grid_joint_candidates_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, nullptr, p, offsets, batch, n_events, motion, cx, cy, cand, n_cand < 1 ? -1 : n_cand,
                              gh, gw, H, W, blur_sigma, objective, 1, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    // the folded images go to ws.Wimg, which a forward-only workspace has no other use for
    return depth_grid_forward<true>(D, ws, taps, batch, objective, obj_param, ws.Wimg, f_out, static_cast<cudaStream_t>(stream));
}

size_t evk_cmax_motion_objective_workspace_bytes(int batch, int H, int W)
{
    if (!evk::batch_limits(batch, 0, H, W, 1)) return 0;
    return evk::batch_obj_carve(nullptr, batch, H, W, (size_t)(H + 1) * (W + 1), nullptr);
}

// The contrast entries and their depth twins share these bodies: rho is the inverse depth of every event, which the
// twins (depth) take for EVK_WARP_CAMERA_MOTION and the others pass as null.
static int cmax_motion_objective(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                 const float *p, const float *rho, const int64_t *offsets, int batch, int64_t n_events,
                                 int warp, const double *params, int K, double cx, double cy, int H, int W, double sigma,
                                 int objective, double obj_param, double *f_out, float *iwe_out, void *workspace,
                                 size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, nullptr, p, rho, depth, offsets, batch, n_events, warp, params, K, cx, cy, H, W,
                         sigma, objective, 1, (size_t)(H + 1) * (W + 1), 0, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !iwe_out)) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc;
    // nonfinite stays zero: a motion sample's non-finite events contribute nothing (model_taps), as in the single window
    EVK_CUDA(batch_obj_zero(ws, batch, npix, 4, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_obj_event_kernel<wt.value, false><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    batch_obj_forward_tail(ws, Hc, Wc, taps, batch, objective, obj_param, iwe_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

static int cmax_motion_objective_grad(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                      const float *p, const float *rho, const int64_t *offsets, int batch,
                                      int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                      int H, int W, double sigma, int objective, double obj_param, const float *iwe,
                                      const float *grad_f, double *grad_params, void *workspace, size_t workspace_bytes,
                                      void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, nullptr, p, rho, depth, offsets, batch, n_events, warp, params, K, cx, cy, H, W,
                         sigma, objective, 1, (size_t)(H + 1) * (W + 1), 0, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_params)) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    EVK_CUDA(cudaMemsetAsync(grad_params, 0, (size_t)batch * K * sizeof(double), st));
    batch_obj_backward_W(ws, iwe, H + 1, W + 1, taps, batch, objective, obj_param, grad_f, st);
    A.Wimg = ws.Wimg;
    A.grad = grad_params;
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_obj_event_kernel<wt.value, true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

static int cmax_motion_candidates(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                  const float *p, const float *rho, const int64_t *offsets, int batch, int64_t n_events,
                                  int warp, const double *cand, int n_cand, int K, double cx, double cy, int H, int W,
                                  double blur_sigma, int objective, double obj_param, double *f_out, void *workspace,
                                  size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, nullptr, p, rho, depth, offsets, batch, n_events, warp, cand, K, cx, cy, H, W,
                         blur_sigma, objective, 1, (size_t)(H + 1) * (W + 1), n_cand < 1 ? -1 : n_cand, workspace,
                         workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, canvases = batch * n_cand;
    // nonfinite stays zero, as in evk_cmax_motion_objective_f32
    EVK_CUDA(batch_obj_zero(ws, canvases, npix, 4, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_seg_cand_kernel<wt.value, false><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    // the folded images go to ws.Wimg, which a forward-only workspace has no other use for
    batch_obj_forward_tail(ws, Hc, Wc, taps, canvases, objective, obj_param, ws.Wimg, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_motion_objective_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                  int batch, int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                  int H, int W, double sigma, int objective, double obj_param, double *f_out, float *iwe_out,
                                  void *workspace, size_t workspace_bytes, void *stream)
{
    return cmax_motion_objective("evk_cmax_motion_objective_f32", false, x, y, t_rel, p, nullptr, offsets, batch, n_events,
                                 warp, params, K, cx, cy, H, W, sigma, objective, obj_param, f_out, iwe_out, workspace,
                                 workspace_bytes, stream);
}

int evk_cmax_motion_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                       int batch, int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                       int H, int W, double sigma, int objective, double obj_param, const float *iwe,
                                       const float *grad_f, double *grad_params, void *workspace, size_t workspace_bytes,
                                       void *stream)
{
    return cmax_motion_objective_grad("evk_cmax_motion_objective_grad_f32", false, x, y, t_rel, p, nullptr, offsets, batch,
                                      n_events, warp, params, K, cx, cy, H, W, sigma, objective, obj_param, iwe, grad_f,
                                      grad_params, workspace, workspace_bytes, stream);
}

size_t evk_cmax_motion_candidates_workspace_bytes(int batch, int n_cand, int H, int W)
{
    if (!evk::batch_limits(batch, n_cand < 1 ? -1 : n_cand, H, W, 1)) return 0;
    return evk::batch_obj_carve(nullptr, batch * n_cand, H, W, (size_t)(H + 1) * (W + 1), nullptr, false);
}

int evk_cmax_motion_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p, const int64_t *offsets,
                                   int batch, int64_t n_events, int warp, const double *cand, int n_cand, int K, double cx,
                                   double cy, int H, int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                   void *workspace, size_t workspace_bytes, void *stream)
{
    return cmax_motion_candidates("evk_cmax_motion_candidates_f32", false, x, y, t_rel, p, nullptr, offsets, batch, n_events,
                                  warp, cand, n_cand, K, cx, cy, H, W, blur_sigma, objective, obj_param, f_out, workspace,
                                  workspace_bytes, stream);
}

size_t evk_cmax_motion_depth_objective_workspace_bytes(int batch, int H, int W)
{
    return evk_cmax_motion_objective_workspace_bytes(batch, H, W);
}

int evk_cmax_motion_depth_objective_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                        const float *inv_depth, const int64_t *offsets, int batch, int64_t n_events,
                                        int warp, const double *params, int K, double cx, double cy, int H, int W,
                                        double sigma, int objective, double obj_param, double *f_out, float *iwe_out,
                                        void *workspace, size_t workspace_bytes, void *stream)
{
    return cmax_motion_objective("evk_cmax_motion_depth_objective_f32", true, x, y, t_rel, p, inv_depth, offsets, batch,
                                 n_events, warp, params, K, cx, cy, H, W, sigma, objective, obj_param, f_out, iwe_out,
                                 workspace, workspace_bytes, stream);
}

int evk_cmax_motion_depth_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                             const float *inv_depth, const int64_t *offsets, int batch,
                                             int64_t n_events, int warp, const double *params, int K, double cx,
                                             double cy, int H, int W, double sigma, int objective, double obj_param,
                                             const float *iwe, const float *grad_f, double *grad_params,
                                             void *workspace, size_t workspace_bytes, void *stream)
{
    return cmax_motion_objective_grad("evk_cmax_motion_depth_objective_grad_f32", true, x, y, t_rel, p, inv_depth, offsets,
                                      batch, n_events, warp, params, K, cx, cy, H, W, sigma, objective, obj_param, iwe,
                                      grad_f, grad_params, workspace, workspace_bytes, stream);
}

size_t evk_cmax_motion_depth_candidates_workspace_bytes(int batch, int n_cand, int H, int W)
{
    return evk_cmax_motion_candidates_workspace_bytes(batch, n_cand, H, W);
}

int evk_cmax_motion_depth_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p,
                                         const float *inv_depth, const int64_t *offsets, int batch, int64_t n_events,
                                         int warp, const double *cand, int n_cand, int K, double cx, double cy, int H,
                                         int W, double blur_sigma, int objective, double obj_param, double *f_out,
                                         void *workspace, size_t workspace_bytes, void *stream)
{
    return cmax_motion_candidates("evk_cmax_motion_depth_candidates_f32", true, x, y, t_rel, p, inv_depth, offsets, batch,
                                  n_events, warp, cand, n_cand, K, cx, cy, H, W, blur_sigma, objective, obj_param, f_out,
                                  workspace, workspace_bytes, stream);
}

size_t evk_cmax_motion_segment_workspace_bytes(int batch, int n_models, int H, int W)
{
    if (!evk::seg_limits(batch, n_models, 0, H, W)) return 0;
    return evk::batch_obj_carve(nullptr, batch * n_models, H, W, (size_t)(H + 1) * (W + 1), nullptr);
}

int evk_cmax_motion_segment_f32(const float *x, const float *y, const float *t_rel, const float *p, const float *weights,
                                int n_models, const int64_t *offsets, int batch, int64_t n_events, int warp, const double *params,
                                int K, double cx, double cy, int H, int W, double sigma, int objective, double obj_param,
                                double *f_out, float *iwe_out, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = motion_seg_setup("evk_cmax_motion_segment_f32", x, y, t_rel, p, weights, n_models, offsets, batch, n_events, warp,
                              params, K, cx, cy, H, W, sigma, objective, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !iwe_out)) { set_error("evk_cmax_motion_segment_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, canvases = batch * n_models;
    // nonfinite stays zero, as in evk_cmax_motion_objective_f32
    EVK_CUDA(batch_obj_zero(ws, canvases, npix, 4, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_model_warp(warp, [&](auto wt) {
            motion_seg_cand_kernel<wt.value, true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    batch_obj_forward_tail(ws, Hc, Wc, taps, canvases, objective, obj_param, iwe_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_motion_segment_grad_f32(const float *x, const float *y, const float *t_rel, const float *p, const float *weights,
                                     int n_models, const int64_t *offsets, int batch, int64_t n_events, int warp,
                                     const double *params, int K, double cx, double cy, int H, int W, double sigma, int objective,
                                     double obj_param, const float *iwe, const float *grad_f, double *grad_params,
                                     float *grad_weights, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = motion_seg_setup("evk_cmax_motion_segment_grad_f32", x, y, t_rel, p, weights, n_models, offsets, batch, n_events,
                              warp, params, K, cx, cy, H, W, sigma, objective, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!iwe || !grad_f || !grad_params)) { set_error("evk_cmax_motion_segment_grad_f32: null array"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, canvases = batch * n_models;
    EVK_CUDA(cudaMemsetAsync(grad_params, 0, (size_t)canvases * K * sizeof(double), st));
    batch_obj_backward_W(ws, iwe, Hc, Wc, taps, canvases, objective, obj_param, grad_f, st);
    if (grad_weights && objective == OBJ_VARIANCE) {
        // the mean of every G_bm (ws.G, just recomputed) for the constant term of the variance's dF/dI
        EVK_CUDA(cudaMemsetAsync(ws.gsums, 0, (size_t)canvases * 8 * sizeof(double), st));
        EVK_CUDA(cudaMemsetAsync(ws.gmax, 0, (size_t)canvases * sizeof(unsigned), st));
        prof_count(1);
        cmax_model_stats_kernel<<<dim3((npix + 255) / 256, 1, canvases), 256, 0, st>>>(ws.G, iwe, npix, objective, obj_param, ws.gsums,
                                                                                        ws.gmax, nullptr, nullptr);
        A.gsums = ws.gsums;
    }
    A.Wimg = ws.Wimg;
    A.grad = grad_params;
    A.grad_f = grad_f;
    A.grad_w = grad_weights;
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        dim3 grid = batch_grid(n_events, batch);
        grid.z = n_models;
        with_model_warp(warp, [&](auto wt) { motion_seg_grad_kernel<wt.value><<<grid, kFlowObjThreads, 0, st>>>(A); });
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_cmax_motion_segment_candidates_workspace_bytes(int batch, int n_models, int n_cand, int H, int W)
{
    if (!evk::seg_limits(batch, n_models, n_cand < 1 ? -1 : n_cand, H, W)) return 0;
    return evk::batch_obj_carve(nullptr, batch * n_models * n_cand, H, W, (size_t)(H + 1) * (W + 1), nullptr, false);
}

int evk_cmax_motion_segment_candidates_f32(const float *x, const float *y, const float *t_rel, const float *p, const float *weights,
                                           int n_models, const int64_t *offsets, int batch, int64_t n_events, int warp,
                                           const double *cand, int n_cand, int K, double cx, double cy, int H, int W,
                                           double blur_sigma, int objective, double obj_param, double *f_out, void *workspace,
                                           size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = motion_seg_setup("evk_cmax_motion_segment_candidates_f32", x, y, t_rel, p, weights, n_models, offsets, batch, n_events,
                              warp, cand, K, cx, cy, H, W, blur_sigma, objective, workspace, workspace_bytes, A, ws, taps,
                              n_cand < 1 ? -1 : n_cand);
    if (rc) return rc;
    if (batch > 0 && !f_out) { set_error("evk_cmax_motion_segment_candidates_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, canvases = batch * n_models * n_cand;
    EVK_CUDA(batch_obj_zero(ws, canvases, npix, 4, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_model_warp(warp, [&](auto wt) {
            motion_seg_cand_kernel<wt.value, true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    batch_obj_forward_tail(ws, Hc, Wc, taps, canvases, objective, obj_param, ws.Wimg, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_cmax_motion_segment_assign_f32(const float *x, const float *y, const float *t_rel, int n_models, const int64_t *offsets,
                                       int batch, int64_t n_events, int warp, const double *params, int K, double cx, double cy,
                                       int H, int W, const float *iwe, double sigma, double eps, float *weights_out,
                                       void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_cmax_motion_segment_assign_f32";
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    // no polarity and no weights enter the assignment: x stands in for both in the shared checks
    int rc = motion_seg_setup(who, x, y, t_rel, x, x, n_models, offsets, batch, n_events, warp, params, K, cx, cy, H, W, sigma,
                              OBJ_VARIANCE, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (!(eps >= 0.0) || !isfinite(eps)) { set_error("%s: eps must be finite and >= 0", who); return EVK_E_ARG; }
    if (batch > 0 && (!iwe || (n_events > 0 && !weights_out))) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    batch_obj_blur(ws, iwe, H + 1, W + 1, taps, batch * n_models, st);
    A.G = ws.G;
    A.eps = eps;
    A.w_out = weights_out;
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_model_warp(warp, [&](auto wt) {
            motion_seg_assign_kernel<wt.value><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_flow_timestamp_objective_workspace_bytes(int batch, int H, int W)
{
    if (!evk::batch_limits(batch, 0, H, W, 2)) return 0;
    return evk::batch_obj_carve(nullptr, 2 * batch, H, W, evk::flow_ts_acc_blocks(H, W), nullptr);
}

int evk_flow_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                     const int64_t *offsets, int batch, int64_t n_events, const float *flow, int H, int W,
                                     double sigma, double *f_out, float *ts_out, float *cnt_out, void *workspace,
                                     size_t workspace_bytes, void *stream)
{
    using namespace evk;
    FlowArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = flow_setup("evk_flow_timestamp_objective_f32", x, y, t_rel, tau, p, offsets, batch, n_events, flow, H, W, sigma, OBJ_SOS,
                        2, flow_ts_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !ts_out || !cnt_out)) { set_error("evk_flow_timestamp_objective_f32: null output"); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, images = 2 * batch;
    EVK_CUDA(batch_obj_zero(ws, images, npix, 8, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        flow_ts_event_kernel<false><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
    }
    ts_obj_forward_tail(ws, Hc, Wc, taps, batch, ts_out, cnt_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_flow_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                          const int64_t *offsets, int batch, int64_t n_events, const float *flow, int H, int W,
                                          double sigma, const float *ts_img, const float *cnt_img, const float *grad_f,
                                          float *grad_flow, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    FlowArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = flow_setup("evk_flow_timestamp_objective_grad_f32", x, y, t_rel, tau, p, offsets, batch, n_events, flow, H, W, sigma,
                        OBJ_SOS, 2, flow_ts_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!ts_img || !cnt_img || !grad_f || !grad_flow)) {
        set_error("evk_flow_timestamp_objective_grad_f32: null array");
        return EVK_E_ARG;
    }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int images = 2 * batch;
    EVK_CUDA(cudaMemsetAsync(ws.acc, 0, (size_t)images * H * W * 4 * sizeof(float), st));
    A.ab = ts_obj_backward_ab(ws, ts_img, cnt_img, H + 1, W + 1, taps, batch, grad_f, st);
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        flow_ts_event_kernel<true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
    }
    prof_count(1);
    flow_obj_grad_fold_kernel<<<grid_simple((int64_t)images * H * W, 256), 256, 0, st>>>(ws.acc, grad_flow, images, H, W);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_motion_timestamp_objective_workspace_bytes(int batch, int H, int W)
{
    if (!evk::batch_limits(batch, 0, H, W, 2)) return 0;
    return evk::batch_obj_carve(nullptr, 2 * batch, H, W, evk::flow_ts_acc_blocks(H, W), nullptr);
}

// The timestamp entries and their depth twins share these bodies, as the contrast entries do.
static int motion_timestamp_objective(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                      const float *tau, const float *p, const float *rho, const int64_t *offsets, int batch,
                                      int64_t n_events, int warp, const double *params, int K, double cx, double cy, int H,
                                      int W, double sigma, double *f_out, float *ts_out, float *cnt_out, void *workspace,
                                      size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, tau, p, rho, depth, offsets, batch, n_events, warp, params, K, cx, cy, H, W, sigma,
                         OBJ_SOS, 2, flow_ts_acc_blocks(H, W), 0, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !ts_out || !cnt_out)) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc, images = 2 * batch;
    // nonfinite stays zero: a non-finite event contributes nothing (model_taps), as in the motion contrast loss
    EVK_CUDA(batch_obj_zero(ws, images, npix, 8, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_ts_event_kernel<wt.value, false><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    ts_obj_forward_tail(ws, Hc, Wc, taps, batch, ts_out, cnt_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

static int motion_timestamp_objective_grad(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                           const float *tau, const float *p, const float *rho, const int64_t *offsets,
                                           int batch, int64_t n_events, int warp, const double *params, int K, double cx,
                                           double cy, int H, int W, double sigma, const float *ts_img, const float *cnt_img,
                                           const float *grad_f, double *grad_params, void *workspace,
                                           size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, tau, p, rho, depth, offsets, batch, n_events, warp, params, K, cx, cy, H, W, sigma,
                         OBJ_SOS, 2, flow_ts_acc_blocks(H, W), 0, workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!ts_img || !cnt_img || !grad_f || !grad_params)) {
        set_error("%s: null array", who);
        return EVK_E_ARG;
    }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    EVK_CUDA(cudaMemsetAsync(grad_params, 0, (size_t)batch * K * sizeof(double), st));
    A.ab = ts_obj_backward_ab(ws, ts_img, cnt_img, H + 1, W + 1, taps, batch, grad_f, st);
    A.grad = grad_params;
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_ts_event_kernel<wt.value, true><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

static int motion_timestamp_candidates(const char *who, bool depth, const float *x, const float *y, const float *t_rel,
                                       const float *tau, const float *p, const float *rho, const int64_t *offsets,
                                       int batch, int64_t n_events, int warp, const double *cand, int n_cand, int K,
                                       double cx, double cy, int H, int W, double blur_sigma, double *f_out,
                                       void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    ModelArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = model_setup(who, x, y, t_rel, tau, p, rho, depth, offsets, batch, n_events, warp, cand, K, cx, cy, H, W,
                         blur_sigma, OBJ_SOS, 2, flow_ts_acc_blocks(H, W), n_cand < 1 ? -1 : n_cand, workspace,
                         workspace_bytes, A, ws, taps);
    if (rc) return rc;
    const int images = 2 * batch * n_cand;
    if (workspace_bytes < motion_ts_cand_bytes(images, H, W)) {
        set_error("%s: 256-byte aligned workspace of %zu bytes required", who, motion_ts_cand_bytes(images, H, W));
        return EVK_E_WORKSPACE;
    }
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int Hc = H + 1, Wc = W + 1, npix = Hc * Wc;
    // nonfinite stays zero, as in evk_motion_timestamp_objective_f32
    EVK_CUDA(batch_obj_zero(ws, images, npix, 8, st));
    if (n_events > 0) {
        ProfScope prof(st);
        prof_count(1);
        with_motion_warp(warp, [&](auto wt) {
            motion_ts_cand_kernel<wt.value><<<batch_grid(n_events, batch), kFlowObjThreads, 0, st>>>(A);
        });
    }
    float *cnt = reinterpret_cast<float *>(static_cast<char *>(workspace) + motion_ts_cand_head(images, H, W));
    ts_obj_forward_tail(ws, Hc, Wc, taps, batch * n_cand, ws.Wimg, cnt, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_motion_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                       const int64_t *offsets, int batch, int64_t n_events, int warp, const double *params,
                                       int K, double cx, double cy, int H, int W, double sigma, double *f_out, float *ts_out,
                                       float *cnt_out, void *workspace, size_t workspace_bytes, void *stream)
{
    return motion_timestamp_objective("evk_motion_timestamp_objective_f32", false, x, y, t_rel, tau, p, nullptr, offsets,
                                      batch, n_events, warp, params, K, cx, cy, H, W, sigma, f_out, ts_out, cnt_out,
                                      workspace, workspace_bytes, stream);
}

int evk_motion_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                            const int64_t *offsets, int batch, int64_t n_events, int warp, const double *params,
                                            int K, double cx, double cy, int H, int W, double sigma, const float *ts_img,
                                            const float *cnt_img, const float *grad_f, double *grad_params, void *workspace,
                                            size_t workspace_bytes, void *stream)
{
    return motion_timestamp_objective_grad("evk_motion_timestamp_objective_grad_f32", false, x, y, t_rel, tau, p, nullptr,
                                           offsets, batch, n_events, warp, params, K, cx, cy, H, W, sigma, ts_img, cnt_img,
                                           grad_f, grad_params, workspace, workspace_bytes, stream);
}

size_t evk_motion_timestamp_candidates_workspace_bytes(int batch, int n_cand, int H, int W)
{
    if (!evk::batch_limits(batch, n_cand < 1 ? -1 : n_cand, H, W, 2)) return 0;
    return evk::motion_ts_cand_bytes(2 * batch * n_cand, H, W);
}

int evk_motion_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                        const int64_t *offsets, int batch, int64_t n_events, int warp, const double *cand,
                                        int n_cand, int K, double cx, double cy, int H, int W, double blur_sigma, double *f_out,
                                        void *workspace, size_t workspace_bytes, void *stream)
{
    return motion_timestamp_candidates("evk_motion_timestamp_candidates_f32", false, x, y, t_rel, tau, p, nullptr, offsets,
                                       batch, n_events, warp, cand, n_cand, K, cx, cy, H, W, blur_sigma, f_out, workspace,
                                       workspace_bytes, stream);
}

size_t evk_motion_timestamp_depth_objective_workspace_bytes(int batch, int H, int W)
{
    return evk_motion_timestamp_objective_workspace_bytes(batch, H, W);
}

int evk_motion_timestamp_depth_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                             const float *p, const float *inv_depth, const int64_t *offsets, int batch,
                                             int64_t n_events, int warp, const double *params, int K, double cx,
                                             double cy, int H, int W, double blur_sigma, double *f_out, float *ts_out,
                                             float *cnt_out, void *workspace, size_t workspace_bytes, void *stream)
{
    return motion_timestamp_objective("evk_motion_timestamp_depth_objective_f32", true, x, y, t_rel, tau, p, inv_depth,
                                      offsets, batch, n_events, warp, params, K, cx, cy, H, W, blur_sigma, f_out, ts_out,
                                      cnt_out, workspace, workspace_bytes, stream);
}

int evk_motion_timestamp_depth_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                                  const float *p, const float *inv_depth, const int64_t *offsets,
                                                  int batch, int64_t n_events, int warp, const double *params, int K,
                                                  double cx, double cy, int H, int W, double blur_sigma,
                                                  const float *ts_img, const float *cnt_img, const float *grad_f,
                                                  double *grad_params, void *workspace, size_t workspace_bytes,
                                                  void *stream)
{
    return motion_timestamp_objective_grad("evk_motion_timestamp_depth_objective_grad_f32", true, x, y, t_rel, tau, p,
                                           inv_depth, offsets, batch, n_events, warp, params, K, cx, cy, H, W, blur_sigma,
                                           ts_img, cnt_img, grad_f, grad_params, workspace, workspace_bytes, stream);
}

size_t evk_motion_timestamp_depth_candidates_workspace_bytes(int batch, int n_cand, int H, int W)
{
    return evk_motion_timestamp_candidates_workspace_bytes(batch, n_cand, H, W);
}

int evk_motion_timestamp_depth_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                              const float *p, const float *inv_depth, const int64_t *offsets,
                                              int batch, int64_t n_events, int warp, const double *cand, int n_cand,
                                              int K, double cx, double cy, int H, int W, double blur_sigma,
                                              double *f_out, void *workspace, size_t workspace_bytes, void *stream)
{
    return motion_timestamp_candidates("evk_motion_timestamp_depth_candidates_f32", true, x, y, t_rel, tau, p, inv_depth,
                                       offsets, batch, n_events, warp, cand, n_cand, K, cx, cy, H, W, blur_sigma, f_out,
                                       workspace, workspace_bytes, stream);
}

size_t evk_grid_flow_timestamp_objective_workspace_bytes(int batch, int gh, int gw, int H, int W)
{
    if (!evk::grid_flow_limits(batch, 0, gh, gw, H, W, 2)) return 0;
    return evk::batch_obj_carve(nullptr, 2 * batch, H, W, evk::flow_ts_acc_blocks(H, W), nullptr);
}

int evk_grid_flow_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                          const int64_t *offsets, int batch, int64_t n_events, const float *grid_flow, int gh,
                                          int gw, int H, int W, double sigma, double *f_out, float *ts_out, float *cnt_out,
                                          void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_grid_flow_timestamp_objective_f32";
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, grid_flow, 0, gh, gw, H, W, sigma, OBJ_SOS, 2,
                             flow_ts_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !ts_out || !cnt_out)) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = grid_flow_event_pass<true>(A, ws, batch, st))) return rc;
    ts_obj_forward_tail(ws, H + 1, W + 1, taps, batch, ts_out, cnt_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_grid_flow_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                               const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                               const float *grid_flow, int gh, int gw, int H, int W, double sigma,
                                               const float *ts_img, const float *cnt_img, const float *grad_f, float *grad_grid,
                                               void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_grid_flow_timestamp_objective_grad_f32";
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, grid_flow, 0, gh, gw, H, W, sigma, OBJ_SOS, 2,
                             flow_ts_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!ts_img || !cnt_img || !grad_f || !grad_grid)) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the f64 node sums live in the accumulator, which the backward has no other use for (ts_obj_backward_ab writes
    // ws.Wimg and ws.wt): 2 batch 2 (H+1)(W+1) 16 B >= batch 2 gh gw 8 B
    A.grad = reinterpret_cast<double *>(ws.acc);
    EVK_CUDA(cudaMemsetAsync(A.grad, 0, (size_t)batch * 2 * gh * gw * sizeof(double), st));
    A.F.ab = ts_obj_backward_ab(ws, ts_img, cnt_img, H + 1, W + 1, taps, batch, grad_f, st);
    return grid_flow_node_grad<true>(A, batch, grad_grid, st);
}

size_t evk_grid_flow_timestamp_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W)
{
    if (!evk::grid_flow_limits(batch, n_cand < 1 ? -1 : n_cand, gh, gw, H, W, 2)) return 0;
    return evk::motion_ts_cand_bytes(2 * batch * n_cand, H, W);
}

int evk_grid_flow_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                           const int64_t *offsets, int batch, int64_t n_events, const float *cand, int n_cand,
                                           int gh, int gw, int H, int W, double blur_sigma, double *f_out, void *workspace,
                                           size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_grid_flow_timestamp_candidates_f32";
    GridArgs A;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = grid_flow_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, cand, n_cand < 1 ? -1 : n_cand, gh, gw, H, W,
                             blur_sigma, OBJ_SOS, 2, flow_ts_acc_blocks(H, W), workspace, workspace_bytes, A, ws, taps);
    if (rc) return rc;
    const int images = 2 * batch * n_cand;
    if (workspace_bytes < motion_ts_cand_bytes(images, H, W)) {
        set_error("%s: 256-byte aligned workspace of %zu bytes required", who, motion_ts_cand_bytes(images, H, W));
        return EVK_E_WORKSPACE;
    }
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = grid_flow_event_pass<true>(A, ws, batch, st))) return rc;
    // T goes to ws.Wimg and C behind the forward-only carve, as in evk_motion_timestamp_candidates_f32
    float *cnt = reinterpret_cast<float *>(static_cast<char *>(workspace) + motion_ts_cand_head(images, H, W));
    ts_obj_forward_tail(ws, H + 1, W + 1, taps, batch * n_cand, ws.Wimg, cnt, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_depth_grid_timestamp_objective_workspace_bytes(int batch, int gh, int gw, int H, int W)
{
    return evk_grid_flow_timestamp_objective_workspace_bytes(batch, gh, gw, H, W);
}

int evk_depth_grid_timestamp_objective_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                           const int64_t *offsets, int batch, int64_t n_events, const double *motion, double cx,
                                           double cy, const float *inv_depth_grid, int gh, int gw, int H, int W, double sigma,
                                           double *f_out, float *ts_out, float *cnt_out, void *workspace,
                                           size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const char *who = "evk_depth_grid_timestamp_objective_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, motion, cx, cy, inv_depth_grid, 0, gh, gw, H,
                              W, sigma, OBJ_SOS, 2, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!f_out || !ts_out || !cnt_out)) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = depth_grid_event_pass<true>(D, ws, batch, st))) return rc;
    ts_obj_forward_tail(ws, H + 1, W + 1, taps, batch, ts_out, cnt_out, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_depth_grid_timestamp_objective_grad_f32(const float *x, const float *y, const float *t_rel, const float *tau,
                                                const float *p, const int64_t *offsets, int batch, int64_t n_events,
                                                const double *motion, double cx, double cy, const float *inv_depth_grid, int gh,
                                                int gw, int H, int W, double sigma, const float *ts_img, const float *cnt_img,
                                                const float *grad_f, float *grad_grid, void *workspace, size_t workspace_bytes,
                                                void *stream)
{
    using namespace evk;
    const char *who = "evk_depth_grid_timestamp_objective_grad_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, motion, cx, cy, inv_depth_grid, 0, gh, gw, H,
                              W, sigma, OBJ_SOS, 2, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    if (batch > 0 && (!ts_img || !cnt_img || !grad_f || !grad_grid)) { set_error("%s: null array", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the f64 node sums live in the accumulator, which the backward has no other use for (ts_obj_backward_ab writes
    // ws.Wimg and ws.wt): 2 batch 2 (H+1)(W+1) 16 B >= batch gh gw 8 B
    D.G.grad = reinterpret_cast<double *>(ws.acc);
    EVK_CUDA(cudaMemsetAsync(D.G.grad, 0, (size_t)batch * gh * gw * sizeof(double), st));
    D.G.F.ab = ts_obj_backward_ab(ws, ts_img, cnt_img, H + 1, W + 1, taps, batch, grad_f, st);
    return depth_grid_node_grad<true>(D, batch, grad_grid, st);
}

size_t evk_depth_grid_timestamp_candidates_workspace_bytes(int batch, int n_cand, int gh, int gw, int H, int W)
{
    return evk_grid_flow_timestamp_candidates_workspace_bytes(batch, n_cand, gh, gw, H, W);
}

int evk_depth_grid_timestamp_candidates_f32(const float *x, const float *y, const float *t_rel, const float *tau, const float *p,
                                            const int64_t *offsets, int batch, int64_t n_events, const double *motion,
                                            double cx, double cy, const float *cand, int n_cand, int gh, int gw, int H, int W,
                                            double blur_sigma, double *f_out, void *workspace, size_t workspace_bytes,
                                            void *stream)
{
    using namespace evk;
    const char *who = "evk_depth_grid_timestamp_candidates_f32";
    DepthGridArgs D;
    BatchObjWorkspace ws;
    BlurTaps taps;
    int rc = depth_grid_setup(who, x, y, t_rel, tau, p, offsets, batch, n_events, motion, cx, cy, cand, n_cand < 1 ? -1 : n_cand,
                              gh, gw, H, W, blur_sigma, OBJ_SOS, 2, workspace, workspace_bytes, D, ws, taps);
    if (rc) return rc;
    const int images = 2 * batch * n_cand;
    if (workspace_bytes < motion_ts_cand_bytes(images, H, W)) {
        set_error("%s: 256-byte aligned workspace of %zu bytes required", who, motion_ts_cand_bytes(images, H, W));
        return EVK_E_WORKSPACE;
    }
    if (batch > 0 && !f_out) { set_error("%s: null output", who); return EVK_E_ARG; }
    if (batch == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = depth_grid_event_pass<true>(D, ws, batch, st))) return rc;
    // T goes to ws.Wimg and C behind the forward-only carve, as in evk_grid_flow_timestamp_candidates_f32
    float *cnt = reinterpret_cast<float *>(static_cast<char *>(workspace) + motion_ts_cand_head(images, H, W));
    ts_obj_forward_tail(ws, H + 1, W + 1, taps, batch * n_cand, ws.Wimg, cnt, f_out, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // extern "C"
