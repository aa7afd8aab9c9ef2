// ccd_inter.cu -- P/B frame reconstruction on sm_90a (SURVEY 8 row a17 / f1).
//
// Replaces the P/B branch of decode_frame (bitstream/decode.py:156-189):
//   apply_global_translation  globalmotion.py:151-160   integer shift, border clamp
//   Warper.forward            warp.py:294-397           TRAINING branch (no 1/64-pel flow rounding),
//                                                       filter_size >= 6: windowed sinc (warp.py:226-268)
//                                                       filter_size 2 / 4: F.grid_sample bilinear / bicubic,
//                                                       border padding, align_corners (warp.py:50-56,314-334)
//   alpha / beta blending     decode.py:171-189
// One thread per pixel; the global shift is folded into the gather indices, so the shifted
// references are never materialised.  Same operation order as oracle/ccoracle.c::warp_sinc
// (coefficients in double -> fp32, fp32 products and sequential sums, no fusion).
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "ccd_detmath.h"
#include "ccd_internal.h"

namespace {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <int N>
__device__ __forceinline__ void sinc_coeffs(float s, float (&c)[N]) {
    const float PIf = 3.14159265358979323846f;
    constexpr int lt = -(N / 2) + 1;
#pragma unroll
    for (int k = 0; k < N; k++) {
        const float arg = __fsub_rn(s, (float)(lt + k));
        const float pa = __fmul_rn(PIf, arg);
        const double win = ccdm_cos((double)__fdiv_rn(pa, (float)N));
        const double sc = (arg == 0.0f) ? 1.0 : __ddiv_rn(ccdm_sin((double)pa), (double)pa);
        c[k] = __fmul_rn((float)win, (float)sc);
    }
}

// Reference planes: plane 0 is [h][w]; planes 1, 2 are [h >> cs][w >> cs] (cs = 1: a YUV 4:2:0 reference, read
// through the nearest x2 up-conversion of convert_420_to_444, io/format/yuv.py:303-316, folded into the gather
// index -- the 4:4:4 copy is never materialised).
struct RefPlanes {
    const float *p[3];
};
__device__ __forceinline__ float ref_at(const RefPlanes &r, int c, int cs, int w, int y, int x) {
    if (c == 0 || cs == 0) return __ldg(r.p[c] + (size_t)y * w + x);
    return __ldg(r.p[c] + (size_t)(y >> 1) * (w >> 1) + (x >> 1));
}

template <int N>
__device__ __forceinline__ void warp_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                           float fy, int x, int y, float (&out)[3]) {
    constexpr int lt = -(N / 2) + 1;
    const float rx = floorf(fx), ry = floorf(fy);
    float cx[N], cy[N];
    sinc_coeffs<N>(__fsub_rn(fx, rx), cx);
    sinc_coeffs<N>(__fsub_rn(fy, ry), cy);
    int xs[N], ys[N];
#pragma unroll
    for (int k = 0; k < N; k++) {
        float nx = __fadd_rn(__fadd_rn((float)x, (float)(lt + k)), rx);
        float ny = __fadd_rn(__fadd_rn((float)y, (float)(lt + k)), ry);
        nx = nx < 0.0f ? 0.0f : (nx > (float)(w - 1) ? (float)(w - 1) : nx);
        ny = ny < 0.0f ? 0.0f : (ny > (float)(h - 1) ? (float)(h - 1) : ny);
        xs[k] = clampi((int)nx + gx, 0, w - 1);
        ys[k] = clampi((int)ny + gy, 0, h - 1);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float col = 0.0f;
#pragma unroll
        for (int i = 0; i < N; i++) {
            float line = 0.0f;
#pragma unroll
            for (int j = 0; j < N; j++) {
                const float t = __fmul_rn(ref_at(ref, c, cs, w, ys[i], xs[j]), cx[j]);
                line = (j == 0) ? t : __fadd_rn(line, t);
            }
            const float t2 = __fmul_rn(line, cy[i]);
            col = (i == 0) ? t2 : __fadd_rn(col, t2);
        }
        out[c] = col;
    }
}

// torch.linspace(-1, 1, n)[i] as PyTorch's CPU kernel evaluates it (see oracle/ccoracle.c::lin_coord)
__device__ __forceinline__ float lin_coord(int n, int i) {
    const float step = __fdiv_rn(2.0f, (float)(n - 1));
    return (i < n / 2) ? __fmaf_rn(step, (float)i, -1.0f) : __fmaf_rn(-step, (float)(n - 1 - i), 1.0f);
}
__device__ __forceinline__ float cubic_near(float x) {
    const float a = __fsub_rn(__fmul_rn(1.25f, x), 2.25f);
    return __fmaf_rn(__fmul_rn(a, x), x, 1.0f);
}
__device__ __forceinline__ float cubic_far(float x) {
    const float a = __fadd_rn(__fmul_rn(-0.75f, x), 3.75f);
    const float b = __fadd_rn(__fmul_rn(a, x), -6.0f);
    return __fadd_rn(__fmul_rn(b, x), 3.0f);
}

// grid_sample(border, align_corners=True) of the globally shifted reference: N == 2 bilinear, N == 4 bicubic.
// Same operation order as oracle/ccoracle.c::warp_grid.
template <int N>
__device__ __forceinline__ void grid_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                           float fy, int x, int y, float (&out)[3]) {
    const float sx = (float)((w - 1.0) / 2.0), sy = (float)((h - 1.0) / 2.0);
    const float g0 = __fadd_rn(lin_coord(w, x), __fdiv_rn(fx, sx)), g1 = __fadd_rn(lin_coord(h, y), __fdiv_rn(fy, sy));
    float ix = __fmul_rn(__fadd_rn(g0, 1.0f), sx), iy = __fmul_rn(__fadd_rn(g1, 1.0f), sy);
    if (N == 2) {
        ix = fminf((float)(w - 1), fmaxf(ix, 0.0f));
        iy = fminf((float)(h - 1), fmaxf(iy, 0.0f));
        const float xw = floorf(ix), yn = floorf(iy);
        const float ww = __fsub_rn(ix, xw), e = __fsub_rn(1.0f, ww), nn = __fsub_rn(iy, yn), s = __fsub_rn(1.0f, nn);
        const float k_nw = __fmul_rn(s, e), k_ne = __fmul_rn(s, ww), k_sw = __fmul_rn(nn, e), k_se = __fmul_rn(nn, ww);
        const int x0 = (int)xw, y0 = (int)yn, x1 = x0 + 1, y1 = y0 + 1;
        const int xa = clampi(x0 + gx, 0, w - 1), xb = clampi((x1 < w ? x1 : w - 1) + gx, 0, w - 1);
        const int ya = clampi(y0 + gy, 0, h - 1), yb = clampi((y1 < h ? y1 : h - 1) + gy, 0, h - 1);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float v00 = ref_at(ref, c, cs, w, ya, xa);
            const float v01 = x1 < w ? ref_at(ref, c, cs, w, ya, xb) : 0.0f;
            const float v10 = y1 < h ? ref_at(ref, c, cs, w, yb, xa) : 0.0f;
            const float v11 = (x1 < w && y1 < h) ? ref_at(ref, c, cs, w, yb, xb) : 0.0f;
            float r = __fmul_rn(v00, k_nw);
            r = __fmaf_rn(v01, k_ne, r);
            r = __fmaf_rn(v10, k_sw, r);
            r = __fmaf_rn(v11, k_se, r);
            out[c] = r;
        }
    } else {
        const float fxx = floorf(ix), fyy = floorf(iy);
        const float tx = __fsub_rn(ix, fxx), ty = __fsub_rn(iy, fyy);
        const float cx[4] = {cubic_far(__fadd_rn(tx, 1.0f)), cubic_near(tx), cubic_near(__fsub_rn(1.0f, tx)),
                             cubic_far(__fsub_rn(2.0f, tx))};
        const float cy[4] = {cubic_far(__fadd_rn(ty, 1.0f)), cubic_near(ty), cubic_near(__fsub_rn(1.0f, ty)),
                             cubic_far(__fsub_rn(2.0f, ty))};
        int xs[4], ys[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float nx = fminf((float)(w - 1), fmaxf(__fadd_rn(fxx, (float)(k - 1)), 0.0f));
            const float ny = fminf((float)(h - 1), fmaxf(__fadd_rn(fyy, (float)(k - 1)), 0.0f));
            xs[k] = clampi((int)nx + gx, 0, w - 1);
            ys[k] = clampi((int)ny + gy, 0, h - 1);
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float rows[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                float r = __fmul_rn(cx[0], ref_at(ref, c, cs, w, ys[i], xs[0]));
                r = __fmaf_rn(cx[1], ref_at(ref, c, cs, w, ys[i], xs[1]), r);
                r = __fmaf_rn(cx[2], ref_at(ref, c, cs, w, ys[i], xs[2]), r);
                r = __fmaf_rn(cx[3], ref_at(ref, c, cs, w, ys[i], xs[3]), r);
                rows[i] = r;
            }
            float a = __fmul_rn(cy[0], rows[0]);
            a = __fmaf_rn(cy[1], rows[1], a);
            a = __fmaf_rn(cy[2], rows[2], a);
            a = __fmaf_rn(cy[3], rows[3], a);
            out[c] = a;
        }
    }
}

template <int N>
__device__ __forceinline__ void predict_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                              float fy, int x, int y, float (&out)[3]) {
    if constexpr (N <= 4)
        grid_pixel<N>(ref, cs, h, w, gx, gy, fx, fy, x, y, out);
    else
        warp_pixel<N>(ref, cs, h, w, gx, gy, fx, fy, x, y, out);
}

// The two predictions of pixel (x, y) and its blending weights (decode.py:171-189): p0, p1 (zero for P), beta (0 for
// P) and the returned alpha, residue channels 4 and 3 plus 0.5, clamped to [0, 1].
template <int N>
__device__ __forceinline__ float predict_refs(const float *__restrict__ residue, const float *__restrict__ motion,
                                              const RefPlanes &ref0, const RefPlanes &ref1, int ref_cs, int h, int w,
                                              int is_b, int g0x, int g0y, int g1x, int g1y, int x, int y,
                                              float (&p0)[3], float (&p1)[3], float &beta) {
    const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
    p1[0] = p1[1] = p1[2] = 0.0f;
    predict_pixel<N>(ref0, ref_cs, h, w, g0x, g0y, motion[i], motion[plane + i], x, y, p0);
    beta = 0.0f;
    if (is_b) {
        predict_pixel<N>(ref1, ref_cs, h, w, g1x, g1y, motion[2 * plane + i], motion[3 * plane + i], x, y, p1);
        beta = __fadd_rn(residue[4 * plane + i], 0.5f);
        beta = clamp01(beta);
    }
    return clamp01(__fadd_rn(residue[3 * plane + i], 0.5f));
}
// the prediction: p0 for P, beta * p0 + (1 - beta) * p1 for B
__device__ __forceinline__ float blend(int is_b, float beta, float p0, float p1) {
    return is_b ? __fadd_rn(__fmul_rn(beta, p0), __fmul_rn(__fsub_rn(1.0f, beta), p1)) : p0;
}

// One thread per pixel; a warp covers a 16 x 2 patch (lane = lx + 16 ly), so that the 2 x 2 chroma blocks of a
// 4:2:0 frame sit inside one warp and the frame tail of decode_frame (bitstream/decode.py:191-206: round ->
// 2 x 2 average of U, V -> clamp -> round) is done with four shuffles instead of a second pass over HBM.
//   M == 0: out[c] = pre-rounding frame (three full planes)
//   M  > 0: out[c] = finished frame on the k / M grid; out_420: U, V planes are [h/2][w/2]
template <int N>
__global__ void __launch_bounds__(128)
    k_inter_predict(const float *__restrict__ residue, const float *__restrict__ motion, RefPlanes ref0, RefPlanes ref1,
                    int ref_cs, int h, int w, int is_b, int g0x, int g0y, int g1x, int g1y, float M, int out_420,
                    float *__restrict__ o0, float *__restrict__ o1, float *__restrict__ o2) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int px = blockIdx.x * 32 + (wrp & 1) * 16 + (lane & 15);
    const int py = blockIdx.y * 4 + (wrp >> 1) * 2 + (lane >> 4);
    const bool inside = px < w && py < h;
    const int x = px < w ? px : w - 1, y = py < h ? py : h - 1;  // every lane computes (shuffles below)
    const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
    float p0[3], p1[3], beta;
    const float alpha = predict_refs<N>(residue, motion, ref0, ref1, ref_cs, h, w, is_b, g0x, g0y, g1x, g1y, x, y, p0,
                                        p1, beta);
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = __fadd_rn(__fmul_rn(alpha, blend(is_b, beta, p0[c], p1[c])), residue[c * plane + i]);
    float *const outp[3] = {o0, o1, o2};
    if (M == 0.0f) {
        if (inside) {
#pragma unroll
            for (int c = 0; c < 3; c++) outp[c][i] = v[c];
        }
        return;
    }
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = quant(v[c], M);
    if (!out_420) {
        if (inside) {
#pragma unroll
            for (int c = 0; c < 3; c++) outp[c][i] = quant(clamp01(v[c]), M);
        }
        return;
    }
    if (inside) o0[i] = quant(clamp01(v[0]), M);
    // 2 x 2 average of the rounded chroma samples, in the order of F.avg_pool2d's reference loop (yuv.py:295)
    const int base = lane & ~17;
#pragma unroll
    for (int c = 1; c < 3; c++) {
        float s = 0.0f;
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 1));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 16));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 17));
        if (lane == base && px + 1 < w && py + 1 < h)
            outp[c][(size_t)(py >> 1) * (w >> 1) + (px >> 1)] = quant(clamp01(__fdiv_rn(s, 4.0f)), M);
    }
}

// Statistics of the P/B prediction (training/test.py:169-199), one thread per pixel of a 32 x 4 tile: p0, p1, beta,
// alpha and pred with exactly the fp32 operations of k_inter_predict, and with a source orig = ks / M (4:2:0 chroma
// read at >> 1, convert_420_to_444) and dummy = ((0 + r0) + r1) / n_refs.  Per-pixel f64 terms, then a fixed-order
// tree over the CTA: one partial per CTA and per sum, added by the host in tile order (the same value on every run).
template <int N>
__global__ void __launch_bounds__(128)
    k_inter_stats(const float *__restrict__ residue, const float *__restrict__ motion, RefPlanes ref0, RefPlanes ref1,
                  int ref_cs, int h, int w, int is_b, int g0x, int g0y, int g1x, int g1y, InterStatsOut o) {
    __shared__ double red[4][128];
    const int t = threadIdx.x;
    const int x = blockIdx.x * 32 + (t & 31), y = blockIdx.y * 4 + (t >> 5);
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    if (x < w && y < h) {
        const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
        float p0[3], p1[3], beta;
        const float alpha = predict_refs<N>(residue, motion, ref0, ref1, ref_cs, h, w, is_b, g0x, g0y, g1x, g1y, x, y,
                                            p0, p1, beta);
        float pred[3];
#pragma unroll
        for (int c = 0; c < 3; c++) pred[c] = blend(is_b, beta, p0[c], p1[c]);
        acc[0] = alpha;
        acc[1] = beta;
        if (o.src) {
            const size_t wc = (size_t)(w >> ref_cs), nc = (size_t)(h >> ref_cs) * wc;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const size_t k = o.src_hwc ? 3 * i + c
                                           : (c == 0 ? i : plane + (c - 1) * nc + (size_t)(y >> ref_cs) * wc + (x >> ref_cs));
                const int ks = source_sample(o.src, o.src_wide, k);
                const float orig = __fdiv_rn((float)ks, o.src_M);
                float dummy = __fadd_rn(0.0f, ref_at(ref0, c, ref_cs, w, y, x));
                if (is_b) dummy = __fadd_rn(dummy, ref_at(ref1, c, ref_cs, w, y, x));
                dummy = __fdiv_rn(dummy, is_b ? 2.0f : 1.0f);
                const float e = __fsub_rn(pred[c], orig), f = __fsub_rn(dummy, orig);
                acc[2] += (double)__fmul_rn(e, e);
                acc[3] += (double)__fmul_rn(f, f);
            }
        }
        if (o.alpha) o.alpha[i] = alpha;
        if (o.beta) o.beta[i] = beta;
        if (o.pred) {
#pragma unroll
            for (int c = 0; c < 3; c++) o.pred[c * plane + i] = pred[c];
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) red[k][t] = acc[k];
    __syncthreads();
    for (int s = 64; s > 0; s >>= 1) {
        if (t < s) {
#pragma unroll
            for (int k = 0; k < 4; k++) red[k][t] += red[k][t + s];
        }
        __syncthreads();
    }
    if (t < 4) o.part[4 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x) + t] = red[t][0];
}

// Motion analysis (DESIGN §4.9), in the 16 x 2 warp patches of k_inter_predict.  Each variant is the reconstruction of
// k_inter_predict with one decoder input overridden (ccdec.h, CcdInterAnalysis), finished by the same frame tail and
// compared with the source as k_frame_dist does: kd = rint(x * M) against ks, per-plane d^2 summed over the warp, one
// integer atomic per warp.  The warp runs three times per reference (decoded flow, global shift only, no flow); the
// alpha / beta / residue variants re-blend the decoded predictions.  Variants are formed one after the other, so only
// one pair of predictions is live at a time.  Flow statistics per reference on the luma pixels: f64 sums in a
// fixed-order CTA tree, max |local| as an integer atomicMax on its f64 bits (non-negative), an integer count outside.
template <int N>
__global__ void __launch_bounds__(128)
    k_inter_analysis(const float *__restrict__ residue, const float *__restrict__ motion, RefPlanes ref0,
                     RefPlanes ref1, int ref_cs, int h, int w, int is_b, int g0x, int g0y, int g1x, int g1y, float M,
                     int out_420, InterAnalysisOut o) {
    __shared__ double red[6][128];
    const int t = threadIdx.x, lane = t & 31, wrp = t >> 5;
    const int px = blockIdx.x * 32 + (wrp & 1) * 16 + (lane & 15);
    const int py = blockIdx.y * 4 + (wrp >> 1) * 2 + (lane >> 4);
    const bool inside = px < w && py < h;
    const int x = px < w ? px : w - 1, y = py < h ? py : h - 1;  // every lane computes (shuffles below)
    const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
    const int gx[2] = {g0x, g1x}, gy[2] = {g0y, g1y};

    // ---- flow statistics of each reference
    unsigned long long bad = ~0ull;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        double acc[3] = {0.0, 0.0, 0.0};
        unsigned long long mbits = 0ull;
        unsigned out = 0u;
        if (inside && (r == 0 || is_b)) {
            const float fx = motion[2 * r * plane + i], fy = motion[(2 * r + 1) * plane + i];
            if (!(isfinite(fx) && isfinite(fy))) bad = (unsigned long long)i;
            const double dx = (double)fx, dy = (double)fy;
            acc[0] = __dadd_rn(dx, (double)gx[r]);
            acc[1] = __dadd_rn(dy, (double)gy[r]);
            acc[2] = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
            mbits = (unsigned long long)__double_as_longlong(acc[2]);
            const double sx = __dadd_rn(__dadd_rn((double)x, (double)gx[r]), dx);
            const double sy = __dadd_rn(__dadd_rn((double)y, (double)gy[r]), dy);
            out = (sx < 0.0 || sx > (double)(w - 1) || sy < 0.0 || sy > (double)(h - 1)) ? 1u : 0u;
            if (o.flow[r]) {
                o.flow[r][i] = __fadd_rn(fx, (float)gx[r]);
                o.flow[r][plane + i] = __fadd_rn(fy, (float)gy[r]);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; k++) red[3 * r + k][t] = acc[k];
        for (int s = 16; s > 0; s >>= 1) {
            const unsigned long long m = __shfl_down_sync(0xffffffffu, mbits, s);
            mbits = m > mbits ? m : mbits;
        }
        out = __reduce_add_sync(0xffffffffu, out);
        if (lane == 0) {
            if (mbits) atomicMax(o.max_bits + r, mbits);
            if (out) atomicAdd(o.outside + r, (unsigned long long)out);
        }
    }
    for (int s = 16; s > 0; s >>= 1) {
        const unsigned long long b = __shfl_down_sync(0xffffffffu, bad, s);
        bad = b < bad ? b : bad;
    }
    if (lane == 0 && bad != ~0ull) atomicMin(o.bad, bad);

    // ---- the source samples of this pixel: luma, and with 4:2:0 the chroma sample of its 2 x 2 block
    const bool own420 = lane == (lane & ~17) && inside;  // the lane that counts a 4:2:0 chroma sample
    int ks[3];
    {
        const size_t wc = (size_t)(w >> ref_cs), nc = (size_t)(h >> ref_cs) * wc;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const size_t k = o.src_hwc ? 3 * i + c
                                       : (c == 0 ? i : plane + (c - 1) * nc + (size_t)(y >> ref_cs) * wc + (x >> ref_cs));
            ks[c] = source_sample(o.src, o.src_wide, k);
        }
    }
    float res[3];
#pragma unroll
    for (int c = 0; c < 3; c++) res[c] = residue[c * plane + i];

    // one variant: alpha * blend(beta, q0, q1) + (residue or 0), the frame tail of k_inter_predict, then the SSE
    auto variant = [&](int v, float alpha, float beta, const float (&q0)[3], const float (&q1)[3], bool with_residue) {
        float s[3];
#pragma unroll
        for (int c = 0; c < 3; c++)
            s[c] = quant(__fadd_rn(__fmul_rn(alpha, blend(is_b, beta, q0[c], q1[c])), with_residue ? res[c] : 0.0f), M);
        unsigned long long e[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float fin;
            bool counts;
            if (c == 0 || !out_420) {
                fin = quant(clamp01(s[c]), M);
                counts = inside;
            } else {  // 2 x 2 average of the rounded chroma samples, as in k_inter_predict
                const int base = lane & ~17;
                float a = 0.0f;
                a = __fadd_rn(a, __shfl_sync(0xffffffffu, s[c], base));
                a = __fadd_rn(a, __shfl_sync(0xffffffffu, s[c], base + 1));
                a = __fadd_rn(a, __shfl_sync(0xffffffffu, s[c], base + 16));
                a = __fadd_rn(a, __shfl_sync(0xffffffffu, s[c], base + 17));
                fin = quant(clamp01(__fdiv_rn(a, 4.0f)), M);
                counts = own420;
            }
            const int d = (int)rintf(__fmul_rn(fin, M)) - ks[c];
            e[c] = counts ? (unsigned long long)((long long)d * d) : 0ull;
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            for (int k = 16; k > 0; k >>= 1) e[c] += __shfl_down_sync(0xffffffffu, e[c], k);
            if (lane == 0 && e[c]) atomicAdd(o.sse + 3 * v + c, e[c]);
        }
    };

    float p0[3], p1[3], beta;
    const float alpha = predict_refs<N>(residue, motion, ref0, ref1, ref_cs, h, w, is_b, g0x, g0y, g1x, g1y, x, y, p0,
                                        p1, beta);
    variant(0, alpha, beta, p0, p1, true);  // decoded
    if (is_b) {
        variant(3, alpha, 1.0f, p0, p1, true);  // ref0_only
        variant(4, alpha, 0.0f, p0, p1, true);  // ref1_only
    }
    variant(5, alpha, beta, p0, p1, false);  // no_residue
    variant(6, 0.0f, beta, p0, p1, true);    // no_prediction
    // no_local_motion: zero local flow, the global shift kept; no_motion: no flow at all (a zero fractional offset
    // does not make the sinc warp a copy, so both go through the warp)
#pragma unroll 1
    for (int z = 0; z < 2; z++) {
        const int s0x = z ? 0 : g0x, s0y = z ? 0 : g0y, s1x = z ? 0 : g1x, s1y = z ? 0 : g1y;
        predict_pixel<N>(ref0, ref_cs, h, w, s0x, s0y, 0.0f, 0.0f, x, y, p0);
        if (is_b) predict_pixel<N>(ref1, ref_cs, h, w, s1x, s1y, 0.0f, 0.0f, x, y, p1);
        variant(1 + z, alpha, beta, p0, p1, true);
    }

    // ---- flow sums: fixed-order tree over the CTA, one partial per CTA and per sum
    __syncthreads();
    for (int s = 64; s > 0; s >>= 1) {
        if (t < s) {
#pragma unroll
            for (int k = 0; k < 6; k++) red[k][t] += red[k][t + s];
        }
        __syncthreads();
    }
    if (t < 6) o.part[6 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x) + t] = red[t][0];
}

// The taps sinc_coeffs<N> gives the warp, one offset per thread (ccd_debug_sinc_coeffs): c[N i + k]
template <int N>
__global__ void k_sinc_coeffs(const float *__restrict__ s, float *__restrict__ c, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float t[N];
    sinc_coeffs<N>(s[i], t);
#pragma unroll
    for (int k = 0; k < N; k++) c[(size_t)N * i + k] = t[k];
}

// One launch of a P/B kernel: launch(std::integral_constant<int, N>, grid, block, ref0, ref1) for the warp filter
// size N of a, on one thread per pixel in CTAs of 128.  Returns -1 for a size no kernel is built for.
template <class F>
int launch_inter(const InterLaunch &a, F &&launch) {
    const dim3 block(128, 1, 1), grid((a.w + 31) / 32, (a.h + 3) / 4, 1);
    RefPlanes r0, r1;
    for (int c = 0; c < 3; c++) {
        r0.p[c] = a.ref0[c];
        r1.p[c] = a.ref1[c] ? a.ref1[c] : a.ref0[c];
    }
    switch (a.filter_size) {
        case 2: if (a.h < 2 || a.w < 2) return -1; launch(std::integral_constant<int, 2>{}, grid, block, r0, r1); break;
        case 4: if (a.h < 2 || a.w < 2) return -1; launch(std::integral_constant<int, 4>{}, grid, block, r0, r1); break;
        case 6: launch(std::integral_constant<int, 6>{}, grid, block, r0, r1); break;
        case 8: launch(std::integral_constant<int, 8>{}, grid, block, r0, r1); break;
        case 10: launch(std::integral_constant<int, 10>{}, grid, block, r0, r1); break;
        case 12: launch(std::integral_constant<int, 12>{}, grid, block, r0, r1); break;
        // the largest size the 4-bit header field can carry (header.py:217)
        case 14: launch(std::integral_constant<int, 14>{}, grid, block, r0, r1); break;
        default: return -1;
    }
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

}  // namespace

int64_t ccd_inter_stats_ctas(int h, int w) { return (int64_t)((w + 31) / 32) * ((h + 3) / 4); }

int ccd_inter_stats_launch(const InterLaunch &a, const InterStatsOut &o, cudaStream_t st) {
    return launch_inter(a, [&](auto n, dim3 grid, dim3 block, const RefPlanes &r0, const RefPlanes &r1) {
        k_inter_stats<decltype(n)::value><<<grid, block, 0, st>>>(a.residue, a.motion, r0, r1, a.ref_cs, a.h, a.w, a.is_b,
                                                                  a.gf[0], a.gf[1], a.gf[2], a.gf[3], o);
    });
}

int ccd_inter_analysis_launch(const InterLaunch &a, const InterAnalysisOut &o, cudaStream_t st) {
    return launch_inter(a, [&](auto n, dim3 grid, dim3 block, const RefPlanes &r0, const RefPlanes &r1) {
        k_inter_analysis<decltype(n)::value><<<grid, block, 0, st>>>(a.residue, a.motion, r0, r1, a.ref_cs, a.h, a.w,
                                                                     a.is_b, a.gf[0], a.gf[1], a.gf[2], a.gf[3], a.M,
                                                                     a.out_420, o);
    });
}

int ccd_inter_launch(const InterLaunch &a, cudaStream_t st) {
    return launch_inter(a, [&](auto n, dim3 grid, dim3 block, const RefPlanes &r0, const RefPlanes &r1) {
        k_inter_predict<decltype(n)::value><<<grid, block, 0, st>>>(a.residue, a.motion, r0, r1, a.ref_cs, a.h, a.w,
                                                                    a.is_b, a.gf[0], a.gf[1], a.gf[2], a.gf[3], a.M,
                                                                    a.out_420, a.out[0], a.out[1], a.out[2]);
    });
}

int ccd_sinc_coeffs(int taps, const float *d_s, float *d_c, size_t n, cudaStream_t st) {
    const unsigned blocks = (unsigned)((n + 127) / 128);
    switch (taps) {
        case 6: k_sinc_coeffs<6><<<blocks, 128, 0, st>>>(d_s, d_c, n); break;
        case 8: k_sinc_coeffs<8><<<blocks, 128, 0, st>>>(d_s, d_c, n); break;
        case 10: k_sinc_coeffs<10><<<blocks, 128, 0, st>>>(d_s, d_c, n); break;
        case 12: k_sinc_coeffs<12><<<blocks, 128, 0, st>>>(d_s, d_c, n); break;
        case 14: k_sinc_coeffs<14><<<blocks, 128, 0, st>>>(d_s, d_c, n); break;
        default: return -1;
    }
    g_ccd_launches++;
    return (int)cudaGetLastError();
}
