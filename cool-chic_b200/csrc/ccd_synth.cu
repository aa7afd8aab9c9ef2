// ccd_synth.cu -- float tail of the Cool-chic decoder on sm_90a: learned upsampling,
// synthesis, final resize, frame quantisation.
//
// Replaces (reference, fp32 PyTorch CPU):
//   core/upsampling.py:189-196   pre-concat conv, TRAIN-mode kron form (zero pad, + x)
//   core/upsampling.py:306-325   transposed conv, TRAIN-mode kron form (replicate pad 4, crop 11)
//   core/upsampling.py:463-500   Upsampling.forward cascade
//   core/synthesis.py:61-76      SynthesisConv2d.forward (replicate pad, conv+bias, +x, ReLU)
//   core/synthesis.py:272-294    Synthesis.forward (trunk + stabiliser, output_transform)
//   component/coolchic.py:187-192 final F.interpolate + crop
//   bitstream/decode.py:191-206  round / 420 average / clamp / round
//
// Canonical fp32 order (identical to oracle/ccoracle.c, so GPU == oracle bit for bit):
// every output is acc = init; for ci, for ky, for kx: acc = fmaf(w, x, acc).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "ccd_detmath.h"
#include "ccd_internal.h"

namespace {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

struct K1d {
    float w[16];
};

__global__ void k_ups_first(const int8_t *__restrict__ lat, size_t n, float *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)lat[i];
}

// hi = conv2d(x, kron(w, w), zero padding k/2) + x      (x = int8 latent as float)
__global__ void k_ups_pre(const int8_t *__restrict__ lat, int h, int w, K1d kw, int k, float *__restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int p = k / 2;
    float acc = 0.0f;
    for (int a = 0; a < k; a++) {
        const int yy = y + a - p;
        if (yy < 0 || yy >= h) continue;
        for (int b = 0; b < k; b++) {
            const int xx = x + b - p;
            if (xx < 0 || xx >= w) continue;
            const float kk = __fmul_rn(kw.w[a], kw.w[b]);
            acc = __fmaf_rn(kk, (float)lat[(size_t)yy * w + xx], acc);
        }
    }
    out[(size_t)y * w + x] = __fadd_rn(acc, (float)lat[(size_t)y * w + x]);
}

// transposed conv stride 2 on the replicate-padded input, cropped (see oracle convt_kron)
__global__ void k_ups_convt(const float *__restrict__ in, int h, int w, K1d kw, int k, float *__restrict__ out,
                            int ht, int wt) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int u = blockIdx.y * blockDim.y + threadIdx.y;
    const int c = blockIdx.z;
    if (v >= wt || u >= ht) return;
    const int P0 = k / 2, C = 2 * P0 - 1 + k / 2;
    const float *src = in + (size_t)c * h * w;
    const int o1 = u + C, o2 = v + C;
    const int i1_lo = (o1 - (k - 1) < 0) ? 0 : (o1 - (k - 1) + 1) / 2, i1_hi = o1 / 2;
    const int i2_lo = (o2 - (k - 1) < 0) ? 0 : (o2 - (k - 1) + 1) / 2, i2_hi = o2 / 2;
    float acc = 0.0f;
    for (int i1 = i1_lo; i1 <= i1_hi; i1++) {
        const int a = o1 - 2 * i1;
        const int r = clampi(i1 - P0, 0, h - 1);
        for (int i2 = i2_lo; i2 <= i2_hi; i2++) {
            const int b = o2 - 2 * i2;
            const int cc = clampi(i2 - P0, 0, w - 1);
            const float kk = __fmul_rn(kw.w[a], kw.w[b]);
            acc = __fmaf_rn(kk, src[(size_t)r * w + cc], acc);
        }
    }
    out[((size_t)c * ht + u) * wt + v] = acc;
}

// One level of the upsampling cascade (Upsampling.forward, upsampling.py:463-500) for the default kernel
// sizes (8-tap transposed conv, 7-tap pre-concatenation conv) in ONE launch: blockIdx.z == 0 filters the
// target grid's own latent (k_ups_pre), z >= 1 upsamples channel z - 1 of the coarser stack (k_ups_convt).
// The separable kernels' 2-D products w[a] * w[b] are formed once on the host (one fp32 multiply each, the
// same value the per-tap __fmul_rn gives); a thread of the transposed part produces a 2 x 2 output block from
// one 5 x 5 clamped input window (25 loads for 64 FMAs).  Accumulation order per output = k_ups_convt / k_ups_pre.
struct UpsLevelParams {
    const int8_t *lat;  // target grid [th][tw]
    const float *in;    // coarser stack [cc][ch][cw]
    float *out;         // [cc + 1][th][tw]
    int cc, ch, cw, th, tw;
    float kt[8][8];     // transposed-conv taps
    float kc[7][7];     // pre-concatenation taps
};
__global__ void __launch_bounds__(256) k_ups_level(UpsLevelParams P) {
    const int th = P.th, tw = P.tw;
    if (blockIdx.z == 0) {
        const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
        if (x >= tw || y >= th) return;
        float acc = 0.0f;
#pragma unroll
        for (int a = 0; a < 7; a++) {
            const int yy = y + a - 3;
#pragma unroll
            for (int b = 0; b < 7; b++) {
                const int xx = x + b - 3;
                if (yy >= 0 && yy < th && xx >= 0 && xx < tw) acc = __fmaf_rn(P.kc[a][b], (float)P.lat[(size_t)yy * tw + xx], acc);
            }
        }
        P.out[(size_t)y * tw + x] = __fadd_rn(acc, (float)P.lat[(size_t)y * tw + x]);
        return;
    }
    // transposed part: output block (2q .. 2q+1, 2s .. 2s+1)
    const int s0 = blockIdx.x * 32 + threadIdx.x, q = blockIdx.y * 8 + threadIdx.y;
    if (2 * s0 >= tw || 2 * q >= th) return;
    const int c = blockIdx.z - 1, h = P.ch, w = P.cw;
    const float *src = P.in + (size_t)c * h * w;
    float win[5][5];
#pragma unroll
    for (int i = 0; i < 5; i++) {
        const float *row = src + (size_t)clampi(q - 2 + i, 0, h - 1) * w;
#pragma unroll
        for (int j = 0; j < 5; j++) win[i][j] = __ldg(row + clampi(s0 - 2 + j, 0, w - 1));
    }
    float *dst = P.out + (size_t)(c + 1) * th * tw;
#pragma unroll
    for (int du = 0; du < 2; du++) {
        const int u = 2 * q + du;
        if (u >= th) continue;
#pragma unroll
        for (int dv = 0; dv < 2; dv++) {
            const int v = 2 * s0 + dv;
            if (v >= tw) continue;
            // u = 2q: input rows q-2 .. q+1 with taps a = 7, 5, 3, 1;  u = 2q+1: rows q-1 .. q+2, a = 6, 4, 2, 0
            float acc = 0.0f;
#pragma unroll
            for (int t1 = 0; t1 < 4; t1++)
#pragma unroll
                for (int t2 = 0; t2 < 4; t2++)
                    acc = __fmaf_rn(P.kt[(1 - du) + 6 - 2 * t1][(1 - dv) + 6 - 2 * t2], win[t1 + du][t2 + dv], acc);
            dst[(size_t)u * tw + v] = acc;
        }
    }
}

// generic SynthesisConv2d: one thread = one pixel, loops over output channels
__global__ void k_syn_layer(const float *__restrict__ in, int h, int w, int cin, int cout, int k, int residual,
                            int relu, const float *__restrict__ wt, const float *__restrict__ bias,
                            float *__restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int p = (k - 1) / 2;
    const size_t plane = (size_t)h * w;
    for (int co = 0; co < cout; co++) {
        float acc = __ldg(bias + co);
        for (int ci = 0; ci < cin; ci++) {
            for (int ky = 0; ky < k; ky++) {
                const int yy = clampi(y + ky - p, 0, h - 1);
                for (int kx = 0; kx < k; kx++) {
                    const int xx = clampi(x + kx - p, 0, w - 1);
                    acc = __fmaf_rn(__ldg(wt + (((size_t)co * cin + ci) * k + ky) * k + kx),
                                    in[ci * plane + (size_t)yy * w + xx], acc);
                }
            }
        }
        if (residual) acc = __fadd_rn(acc, in[co * plane + (size_t)y * w + x]);
        if (relu) acc = fmaxf(acc, 0.0f);
        out[co * plane + (size_t)y * w + x] = acc;
    }
}

// two fused 1x1 layers (cin -> chid -> cout), hidden activations stay in registers.
// Same summation order as two sequential generic layers.
template <int CIN_MAX, int COUT_MAX>
__global__ void k_syn_pw2(const float *__restrict__ in, size_t plane, int cin, int chid, int cout, int relu0,
                          int relu1, const float *__restrict__ w0, const float *__restrict__ b0,
                          const float *__restrict__ w1, const float *__restrict__ b1, float *__restrict__ out) {
    extern __shared__ float s_w[];
    float *sw0 = s_w;                   // [chid][cin]
    float *sb0 = sw0 + chid * cin;      // [chid]
    float *sw1 = sb0 + chid;            // [cout][chid]
    float *sb1 = sw1 + cout * chid;     // [cout]
    for (int i = threadIdx.x; i < chid * cin; i += blockDim.x) sw0[i] = w0[i];
    for (int i = threadIdx.x; i < chid; i += blockDim.x) sb0[i] = b0[i];
    for (int i = threadIdx.x; i < cout * chid; i += blockDim.x) sw1[i] = w1[i];
    for (int i = threadIdx.x; i < cout; i += blockDim.x) sb1[i] = b1[i];
    __syncthreads();
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= plane) return;
    float x[CIN_MAX], o[COUT_MAX];
#pragma unroll
    for (int i = 0; i < CIN_MAX; i++) x[i] = (i < cin) ? in[(size_t)i * plane + p] : 0.0f;
#pragma unroll
    for (int c = 0; c < COUT_MAX; c++) o[c] = (c < cout) ? sb1[c] : 0.0f;
    for (int hcn = 0; hcn < chid; hcn++) {
        float a = sb0[hcn];
#pragma unroll
        for (int i = 0; i < CIN_MAX; i++)
            if (i < cin) a = __fmaf_rn(sw0[hcn * cin + i], x[i], a);
        if (relu0) a = fmaxf(a, 0.0f);
#pragma unroll
        for (int c = 0; c < COUT_MAX; c++)
            if (c < cout) o[c] = __fmaf_rn(sw1[c * chid + hcn], a, o[c]);
    }
#pragma unroll
    for (int c = 0; c < COUT_MAX; c++)
        if (c < cout) out[(size_t)c * plane + p] = relu1 ? fmaxf(o[c], 0.0f) : o[c];
}

// ---------------------------------------------------------------------------------------------------
// Fused synthesis (core/synthesis.py:272-294) for the architecture family every Cool-chic preset uses:
//   [1x1 cin -> hid (relu?)] [1x1 hid -> C (relu?)] then 0, 1 or 2 3x3 layers C -> C (residual? relu?)
//   + linear stabiliser (1x1 on the dense input) + output transform (1x1 C -> C).
// One CTA = one 32 x 16 output tile.  Stage A evaluates the two 1x1 layers on the tile plus a halo of one
// pixel per 3x3 layer (three positions per thread share each weight fetch), the 3x3 layers go from shared
// memory to shared memory, the stabiliser / residual adds / output transform happen in registers, and only
// the final C planes are written: the dense latent is read once and nothing else touches HBM.
// Replicate padding = every stage evaluates out-of-frame positions at their clamped coordinates.
// Same fp32 operation order per output as the unfused kernels (and oracle/ccoracle.c::syn_conv), so the
// result is bit-identical.
struct SynFusedParams {
    const float *in;    // dense latent [cin][h][w]
    float *out;         // [C][h][w]
    int h, w, cin, hid, n3;            // n3: number of 3x3 layers (0..2)
    int relu0, relu1, res3[2], relu3[2];
    int stab_in;                       // 0: no stabiliser
    const float *w0, *b0, *w1, *b1;    // [hid][cin], [hid], [C][hid], [C]
    const float *w3[2], *b3[2];        // [C][C][3][3], [C]
    const float *ws, *bs, *wo, *bo;    // [C][stab_in], [C], [C][C], [C]
};
constexpr int SF_TW = 32, SF_TH = 16, SF_THREADS = 256;

template <int CINP, int C>
__global__ void __launch_bounds__(SF_THREADS) k_syn_fused(SynFusedParams P) {
    extern __shared__ __align__(16) float sf_smem[];
    const int n3 = P.n3, hid = P.hid, cin = P.cin;
    const int RW = SF_TW + 2 * n3, RH = SF_TH + 2 * n3;  // stage-A region
    // shared memory: weights, then region buffers
    float *sw0 = sf_smem;                    // [hid][CINP]
    float *sb0 = sw0 + hid * CINP;           // [hid]
    float *sw1 = sb0 + hid;                  // [hid][4*ceil(C/4)]  (transposed: one vector load per hidden unit)
    constexpr int CP = (C + 3) & ~3;
    float *sb1 = sw1 + hid * CP;             // [CP]
    float *sw3 = sb1 + CP;                   // [2][C][C][9]
    float *sb3 = sw3 + 2 * C * C * 9;        // [2][CP]
    float *sws = sb3 + 2 * CP;               // [C][CINP]
    float *sbs = sws + C * CINP;             // [CP]
    float *swo = sbs + CP;                   // [C][CP]
    float *sbo = swo + C * CP;               // [CP]
    float *bufA = sbo + CP;                  // [C][RH][RW]
    float *bufB = bufA + C * RH * RW;        // [C][RH-2][RW-2]   (n3 == 2)
    float *sstab = bufB + (n3 == 2 ? C * (RH - 2) * (RW - 2) : 0);  // [C][SF_TH][SF_TW]
    const int tid = threadIdx.x;
    for (int i = tid; i < hid * CINP; i += SF_THREADS) {
        const int hh = i / CINP, ci = i - hh * CINP;
        sw0[i] = ci < cin ? P.w0[hh * cin + ci] : 0.0f;
    }
    for (int i = tid; i < hid; i += SF_THREADS) sb0[i] = P.b0[i];
    for (int i = tid; i < hid * CP; i += SF_THREADS) {
        const int hh = i / CP, c = i - hh * CP;
        sw1[i] = c < C ? P.w1[c * hid + hh] : 0.0f;
    }
    for (int i = tid; i < CP; i += SF_THREADS) {
        sb1[i] = i < C ? P.b1[i] : 0.0f;
        sbs[i] = (i < C && P.stab_in) ? P.bs[i] : 0.0f;
        sbo[i] = i < C ? P.bo[i] : 0.0f;
        for (int l = 0; l < 2; l++) sb3[l * CP + i] = (i < C && l < n3) ? P.b3[l][i] : 0.0f;
    }
    for (int l = 0; l < n3; l++)
        for (int i = tid; i < C * C * 9; i += SF_THREADS) sw3[l * C * C * 9 + i] = P.w3[l][i];
    for (int i = tid; i < C * CINP; i += SF_THREADS) {
        const int c = i / CINP, ci = i - c * CINP;
        sws[i] = (ci < P.stab_in) ? P.ws[c * P.stab_in + ci] : 0.0f;
    }
    for (int i = tid; i < C * CP; i += SF_THREADS) {
        const int c = i / CP, k = i - c * CP;
        swo[i] = k < C ? P.wo[c * C + k] : 0.0f;
    }
    __syncthreads();

    const int x0 = blockIdx.x * SF_TW, y0 = blockIdx.y * SF_TH;
    const int H = P.h, W = P.w;
    const size_t plane = (size_t)H * W;
    // ---- stage A: two 1x1 layers (+ stabiliser on the tile itself) on RH x RW positions, 3 per thread
    const int nA = RH * RW;
    for (int base = 0; base < nA; base += 3 * SF_THREADS) {
        float x[3][CINP], o[3][C];
        int pos[3];
#pragma unroll
        for (int q = 0; q < 3; q++) {
            const int pp = base + q * SF_THREADS + tid;
            pos[q] = pp;
            const int py = pp / RW, px = pp - py * RW;
            const int gy = clampi(y0 - n3 + py, 0, H - 1), gx = clampi(x0 - n3 + px, 0, W - 1);
            const float *src = P.in + (size_t)gy * W + gx;
#pragma unroll
            for (int ci = 0; ci < CINP; ci++) x[q][ci] = (pp < nA && ci < cin) ? __ldg(src + (size_t)ci * plane) : 0.0f;
#pragma unroll
            for (int c = 0; c < C; c++) o[q][c] = sb1[c];
        }
        for (int hh = 0; hh < hid; hh++) {
            float wv[CINP];
#pragma unroll
            for (int v = 0; v < CINP / 4; v++) {
                const float4 t = *reinterpret_cast<const float4 *>(sw0 + hh * CINP + 4 * v);
                wv[4 * v] = t.x; wv[4 * v + 1] = t.y; wv[4 * v + 2] = t.z; wv[4 * v + 3] = t.w;
            }
            float w1v[CP];
#pragma unroll
            for (int v = 0; v < CP / 4; v++) {
                const float4 t = *reinterpret_cast<const float4 *>(sw1 + hh * CP + 4 * v);
                w1v[4 * v] = t.x; w1v[4 * v + 1] = t.y; w1v[4 * v + 2] = t.z; w1v[4 * v + 3] = t.w;
            }
            const float bb = sb0[hh];
#pragma unroll
            for (int q = 0; q < 3; q++) {
                float a = bb;
#pragma unroll
                for (int ci = 0; ci < CINP; ci++)
                    if (ci < cin) a = __fmaf_rn(wv[ci], x[q][ci], a);
                if (P.relu0) a = fmaxf(a, 0.0f);
#pragma unroll
                for (int c = 0; c < C; c++) o[q][c] = __fmaf_rn(w1v[c], a, o[q][c]);
            }
        }
#pragma unroll
        for (int q = 0; q < 3; q++) {
            if (pos[q] >= nA) continue;
            const int py = pos[q] / RW, px = pos[q] - py * RW;
#pragma unroll
            for (int c = 0; c < C; c++) bufA[(c * RH + py) * RW + px] = P.relu1 ? fmaxf(o[q][c], 0.0f) : o[q][c];
            // stabiliser (synthesis.py:286-289) for positions of the tile itself
            const int ty = py - n3, tx = px - n3;
            if (P.stab_in && ty >= 0 && ty < SF_TH && tx >= 0 && tx < SF_TW) {
#pragma unroll
                for (int c = 0; c < C; c++) {
                    float a = sbs[c];
#pragma unroll
                    for (int ci = 0; ci < CINP; ci++)
                        if (ci < P.stab_in) a = __fmaf_rn(sws[c * CINP + ci], x[q][ci], a);
                    sstab[(c * SF_TH + ty) * SF_TW + tx] = a;
                }
            }
        }
    }
    __syncthreads();
    // ---- 3x3 layers, shared memory -> shared memory (the last one -> registers -> output)
    const float *cur = bufA;
    int cw = RW, chh = RH, off = n3;  // current buffer geometry; off = its halo w.r.t. the tile
    for (int l = 0; l < n3 - 1; l++) {
        // intermediate 3x3 layer on the region shrunk by one pixel
        const int ow = cw - 2, oh = chh - 2;
        const float *wl = sw3 + l * C * C * 9;
        for (int pp = tid; pp < ow * oh; pp += SF_THREADS) {
            const int py = pp / ow, px = pp - py * ow;
            // this position in frame coordinates, clamped (replicate padding of the NEXT layer), then back
            // to buffer coordinates of `cur`
            const int gy = clampi(y0 - (off - 1) + py, 0, H - 1), gx = clampi(x0 - (off - 1) + px, 0, W - 1);
            const int by = gy - (y0 - off), bx = gx - (x0 - off);
            float acc[C];
#pragma unroll
            for (int co = 0; co < C; co++) acc[co] = sb3[l * CP + co];
#pragma unroll
            for (int ci = 0; ci < C; ci++)
#pragma unroll
                for (int ky = 0; ky < 3; ky++)
#pragma unroll
                    for (int kx = 0; kx < 3; kx++) {
                        const float v = cur[(ci * chh + by + ky - 1) * cw + bx + kx - 1];
#pragma unroll
                        for (int co = 0; co < C; co++) acc[co] = __fmaf_rn(wl[((co * C + ci) * 3 + ky) * 3 + kx], v, acc[co]);
                    }
#pragma unroll
            for (int co = 0; co < C; co++) {
                float a = acc[co];
                if (P.res3[l]) a = __fadd_rn(a, cur[(co * chh + by) * cw + bx]);
                if (P.relu3[l]) a = fmaxf(a, 0.0f);
                bufB[(co * oh + py) * ow + px] = a;
            }
        }
        __syncthreads();
        cur = bufB;
        cw = ow;
        chh = oh;
        off -= 1;
    }
    // ---- last stage on the tile: last 3x3 layer (if any), + stabiliser, output transform, store
    for (int pp = tid; pp < SF_TW * SF_TH; pp += SF_THREADS) {
        const int ty = pp / SF_TW, tx = pp - ty * SF_TW;
        const int gy = y0 + ty, gx = x0 + tx;
        if (gy >= H || gx >= W) continue;
        const int by = ty + off, bx = tx + off;
        float t[C];
        if (n3 > 0) {
            const int l = n3 - 1;
            const float *wl = sw3 + l * C * C * 9;
#pragma unroll
            for (int co = 0; co < C; co++) t[co] = sb3[l * CP + co];
#pragma unroll
            for (int ci = 0; ci < C; ci++)
#pragma unroll
                for (int ky = 0; ky < 3; ky++)
#pragma unroll
                    for (int kx = 0; kx < 3; kx++) {
                        const float v = cur[(ci * chh + by + ky - 1) * cw + bx + kx - 1];
#pragma unroll
                        for (int co = 0; co < C; co++) t[co] = __fmaf_rn(wl[((co * C + ci) * 3 + ky) * 3 + kx], v, t[co]);
                    }
#pragma unroll
            for (int co = 0; co < C; co++) {
                if (P.res3[l]) t[co] = __fadd_rn(t[co], cur[(co * chh + by) * cw + bx]);
                if (P.relu3[l]) t[co] = fmaxf(t[co], 0.0f);
            }
        } else {
#pragma unroll
            for (int co = 0; co < C; co++) t[co] = cur[(co * chh + by) * cw + bx];
        }
        if (P.stab_in) {
#pragma unroll
            for (int co = 0; co < C; co++) t[co] = __fadd_rn(t[co], sstab[(co * SF_TH + ty) * SF_TW + tx]);
        }
#pragma unroll
        for (int co = 0; co < C; co++) {
            float a = sbo[co];
#pragma unroll
            for (int ci = 0; ci < C; ci++) a = __fmaf_rn(swo[co * CP + ci], t[ci], a);
            P.out[(size_t)co * plane + (size_t)gy * W + gx] = a;
        }
    }
}

// ===================================================================================================
// Batched float tail (BASELINE configs[2] / [4]: many streams in one call).
//
//   k_ups_level_b : one level of the cascade for ALL streams of a group in one launch
//                   (blockIdx.z = stream * planes + plane)
//   k_tail_syn    : the LAST cascade level + the whole synthesis + the frame tail in one kernel.  The dense
//                   latent at image resolution (7 fp32 planes, 28 B / pixel written and read back by the
//                   unfused path) is never materialised: a CTA stages the int8 tile of the finest grid
//                   (zero padding = TMA out-of-bounds fill) and the tile of the half-resolution stack in shared
//                   memory -- with TMA (cp.async.bulk.tensor + mbarrier) when the row pitches allow it -- and
//                   evaluates the 7x7 pre-concatenation conv and the 8x8 stride-2 transposed conv on the fly
//                   for every position of the synthesis region.  Epilogue: output transform, then optionally
//                   decode_frame's round / (4:2:0 average) / clamp / round (bitstream/decode.py:191-206).
// Every output keeps the canonical fp32 operation order of the unfused kernels (bit-identical, tested).
// ===================================================================================================
struct UpsLevelJob {
    const int8_t *lat;  // target grid [th][tw]
    const float *in;    // coarser stack [cc][ch][cw] (fp32) ...
    const int8_t *in8;  // ... or, for the first level, the coarsest latent grid itself (cc == 1)
    float *out;         // [cc + 1][th][tw]
    int cc, ch, cw, th, tw;
    float kt[8][8];     // transposed-conv taps
    float kc[7][7];     // pre-concatenation taps
};
__global__ void __launch_bounds__(256) k_ups_level_b(const UpsLevelJob *__restrict__ jobs, int planes) {
    const int job = blockIdx.z / planes, plane = blockIdx.z - job * planes;
    const UpsLevelJob &P = jobs[job];
    if (plane > P.cc) return;
    const int th = P.th, tw = P.tw;
    if (plane == 0) {
        const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
        if (x >= tw || y >= th) return;
        float acc = 0.0f;
#pragma unroll
        for (int a = 0; a < 7; a++) {
            const int yy = y + a - 3;
#pragma unroll
            for (int b = 0; b < 7; b++) {
                const int xx = x + b - 3;
                if (yy >= 0 && yy < th && xx >= 0 && xx < tw) acc = __fmaf_rn(P.kc[a][b], (float)P.lat[(size_t)yy * tw + xx], acc);
            }
        }
        P.out[(size_t)y * tw + x] = __fadd_rn(acc, (float)P.lat[(size_t)y * tw + x]);
        return;
    }
    const int s0 = blockIdx.x * 32 + threadIdx.x, q = blockIdx.y * 8 + threadIdx.y;
    if (2 * s0 >= tw || 2 * q >= th) return;
    const int c = plane - 1, h = P.ch, w = P.cw;
    float win[5][5];
    if (P.in8) {
        const int8_t *src = P.in8 + (size_t)c * h * w;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            const int8_t *row = src + (size_t)clampi(q - 2 + i, 0, h - 1) * w;
#pragma unroll
            for (int j = 0; j < 5; j++) win[i][j] = (float)row[clampi(s0 - 2 + j, 0, w - 1)];
        }
    } else {
        const float *src = P.in + (size_t)c * h * w;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            const float *row = src + (size_t)clampi(q - 2 + i, 0, h - 1) * w;
#pragma unroll
            for (int j = 0; j < 5; j++) win[i][j] = __ldg(row + clampi(s0 - 2 + j, 0, w - 1));
        }
    }
    float *dst = P.out + (size_t)(c + 1) * th * tw;
#pragma unroll
    for (int du = 0; du < 2; du++) {
        const int u = 2 * q + du;
        if (u >= th) continue;
#pragma unroll
        for (int dv = 0; dv < 2; dv++) {
            const int v = 2 * s0 + dv;
            if (v >= tw) continue;
            float acc = 0.0f;
#pragma unroll
            for (int t1 = 0; t1 < 4; t1++)
#pragma unroll
                for (int t2 = 0; t2 < 4; t2++)
                    acc = __fmaf_rn(P.kt[(1 - du) + 6 - 2 * t1][(1 - dv) + 6 - 2 * t2], win[t1 + du][t2 + dv], acc);
            dst[(size_t)u * tw + v] = acc;
        }
    }
}

struct alignas(64) TailSynJob {
    unsigned char tmap_lat[128];  // CUtensorMap: finest latent grid, uint8 [h][w], box LW x LH
    unsigned char tmap_stk[128];  // CUtensorMap: coarser stack, fp32 [cc][ch][cw], box SW x SH x cc
    const int8_t *lat;            // finest grid [h][w]
    const float *stk;             // coarser stack [cc][ch][cw] (cc = cin - 1), already upsampled to (ch, cw)
    const int8_t *stk8;           // ... or the coarsest latent itself when only two grids exist (cc == 1)
    float *out[3 + 2];            // output planes (C <= 5)
    int h, w, ch, cw, cin, hid, n3;
    int relu0, relu1, res3[2], relu3[2];
    int stab_in;
    int use_tma;                  // 1: tiles staged with TMA (the descriptors above), 0: plain loads
    int finish;                   // 0: raw synthesis output; 1: frame tail, three full planes; 2: frame tail 4:2:0
    float M;                      // 2^bitdepth - 1
    const float *w0, *b0, *w1, *b1;
    const float *w3[2], *b3[2];
    const float *ws, *bs, *wo, *bo;
    float kt[8][8], kc[7][7];
};
// (TMA needs the box to start on a 16-byte boundary in the innermost dimension: the tile origins are rounded down
// to a multiple of 16 int8 / 4 fp32 columns and the boxes widened accordingly)
__host__ __device__ inline int ts_lw(int n3) { return (SF_TW + 2 * n3 + 6 + 15 + 15) & ~15; }
__host__ __device__ inline int ts_lh(int n3) { return SF_TH + 2 * n3 + 6; }
__host__ __device__ inline int ts_sw(int n3) { return ((SF_TW + 2 * n3) / 2 + 5 + 3 + 3) & ~3; }
__host__ __device__ inline int ts_sh(int n3) { return (SF_TH + 2 * n3) / 2 + 5; }

// ---------------------------------------------------------------------------------------------------------------
// k_tail_syn (see the top of this section), laid out for instruction efficiency:
//   * the halo of the stage-A region is rounded up to an even number of pixels, so that the region starts on even
//     frame coordinates and stage A works on 2 x 2 QUADS with compile-time parities: the 8x8 stride-2 transposed
//     conv reads ONE 5 x 5 window per channel for its four outputs, its taps come as 16 vector loads (re-laid
//     [du][t1][dv][t2]); the 7x7 pre-concatenation conv slides over 8 rows of 8 values (converted to fp32 once per
//     tile); the two 1x1 layers share every weight fetch between the four positions;
//   * out-of-frame positions of the region (replicate padding of the 3x3 layers) are copies of the clamped
//     position's values (the 1x1 layers are pointwise), filled by a fix-up pass on border tiles only;
//   * the 3x3 layers evaluate two horizontally adjacent outputs per thread from one 3 x 4 window per channel, their
//     weights re-laid [ci][ky][kx][co] (one vector load per tap); stores are 64-bit.
// Every output keeps its canonical accumulation order: bit-identical to k_syn_fused and the oracle.
__host__ __device__ inline int ts_n3e(int n3) { return (n3 + 1) & ~1; }
constexpr int TS_THREADS = 192;  // 180 quads per 32 x 16 tile with a 2-pixel halo; three CTAs per SM

template <int CINP, int C>
__global__ void __launch_bounds__(TS_THREADS, 3) k_tail_syn(const TailSynJob *__restrict__ jobs) {
    extern __shared__ __align__(128) unsigned char ts_raw[];
    const TailSynJob &P = jobs[blockIdx.z];
    const int H = P.h, W = P.w;
    const int x0 = blockIdx.x * SF_TW, y0 = blockIdx.y * SF_TH;
    if (x0 >= W || y0 >= H) return;
    const int n3 = P.n3, n3e = ts_n3e(n3), hid = P.hid, cin = P.cin, cc = cin - 1;
    const int RW = SF_TW + 2 * n3e, RH = SF_TH + 2 * n3e;
    const int LW = ts_lw(n3e), LH = ts_lh(n3e), SW = ts_sw(n3e), SH = ts_sh(n3e);
    constexpr int CP = (C + 3) & ~3;  // output channels padded to a multiple of 4 (vector loads of weights)
    uint64_t *bar = reinterpret_cast<uint64_t *>(ts_raw);
    int8_t *Lt = reinterpret_cast<int8_t *>(ts_raw + 128);                          // [LH][LW] int8 (TMA destination)
    float *St = reinterpret_cast<float *>(ts_raw + 128 + ((LW * LH + 127) & ~127)); // [cc][SH][SW]
    float *Lf = St + ((cc * SH * SW + 31) & ~31);  // [LH][LW] the latent tile as fp32
    float *sw0 = Lf + LW * LH;               // [hid][CINP]
    float *sb0 = sw0 + hid * CINP;
    float *sw1 = sb0 + ((hid + 3) & ~3);     // [hid][CP]
    float *sb1 = sw1 + hid * CP;
    float *sw3 = sb1 + CP;                   // [2][C][3][3][CP]
    float *sb3 = sw3 + 2 * C * 9 * CP;
    float *sws = sb3 + 2 * CP;               // [C][CINP]
    float *sbs = sws + C * CINP;
    float *swo = sbs + CP;                   // [C][CP]
    float *sbo = swo + C * CP;
    float *skt = sbo + CP;                   // [2 du][4 t1][2 dv][4 t2]
    float *skc = skt + 64;                   // [7][8] (rows padded)
    float *bufA = skc + 56;                  // [C][RH][RW]
    float *bufB = bufA + C * RH * RW;        // [C][RH-2][RW-2]   (n3 == 2)
    float *sstab = bufB + (n3 == 2 ? C * (RH - 2) * (RW - 2) : 0);  // [C][SF_TH][SF_TW]
    const int tid = threadIdx.x;
    const int Y0 = y0 - n3e, X0 = x0 - n3e;                 // stage-A region origin (even frame coordinates)
    const int ly0 = Y0 - 3, lx0 = (X0 - 3) & ~15;           // latent tile (16-byte aligned start)
    const int sy0 = ((Y0 < 0 ? 0 : Y0) >> 1) - 2, sx0 = (((X0 < 0 ? 0 : X0) >> 1) - 2) & ~3;  // stack tile
    const int ch = P.ch, cw = P.cw;
    // ---- stage 0: tiles -> shared memory
    if (P.use_tma) {
        const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
        if (tid == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (tid == 0) {
            const uint32_t bytes = (uint32_t)(LW * LH + cc * SH * SW * 4);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
            const uint64_t tm0 = reinterpret_cast<uint64_t>(P.tmap_lat), tm1 = reinterpret_cast<uint64_t>(P.tmap_stk);
            // the descriptors were written by the host into global memory: fence before their first use
            asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(tm0) : "memory");
            asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(tm1) : "memory");
            asm volatile(
                "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                ::"r"((uint32_t)__cvta_generic_to_shared(Lt)), "l"(tm0), "r"(lx0), "r"(ly0), "r"(bar_a)
                : "memory");
            asm volatile(
                "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                ::"r"((uint32_t)__cvta_generic_to_shared(St)), "l"(tm1), "r"(sx0), "r"(sy0), "r"(0), "r"(bar_a)
                : "memory");
        }
    } else {
        for (int i = tid; i < LW * LH; i += TS_THREADS) {
            const int r = i / LW, c = i - r * LW;
            const int gy = ly0 + r, gx = lx0 + c;
            Lf[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? (float)P.lat[(size_t)gy * W + gx] : 0.0f;
        }
        for (int i = tid; i < cc * SH * SW; i += TS_THREADS) {
            const int c = i / (SH * SW), rem = i - c * SH * SW, r = rem / SW, col = rem - r * SW;
            const int gy = sy0 + r, gx = sx0 + col;
            float v = 0.0f;
            if (gy >= 0 && gy < ch && gx >= 0 && gx < cw)
                v = P.stk8 ? (float)P.stk8[((size_t)c * ch + gy) * cw + gx] : __ldg(P.stk + ((size_t)c * ch + gy) * cw + gx);
            St[i] = v;
        }
    }
    // ---- weights (overlaps the bulk copies)
    for (int i = tid; i < hid * CINP; i += TS_THREADS) {
        const int hh = i / CINP, ci = i - hh * CINP;
        sw0[i] = ci < cin ? P.w0[hh * cin + ci] : 0.0f;
    }
    for (int i = tid; i < hid; i += TS_THREADS) sb0[i] = P.b0[i];
    for (int i = tid; i < hid * CP; i += TS_THREADS) {
        const int hh = i / CP, c = i - hh * CP;
        sw1[i] = c < C ? P.w1[c * hid + hh] : 0.0f;
    }
    for (int i = tid; i < CP; i += TS_THREADS) {
        sb1[i] = i < C ? P.b1[i] : 0.0f;
        sbs[i] = (i < C && P.stab_in) ? P.bs[i] : 0.0f;
        sbo[i] = i < C ? P.bo[i] : 0.0f;
        for (int l = 0; l < 2; l++) sb3[l * CP + i] = (i < C && l < n3) ? P.b3[l][i] : 0.0f;
    }
    for (int l = 0; l < n3; l++)
        for (int i = tid; i < C * 9 * CP; i += TS_THREADS) {
            const int co = i % CP, t = i / CP;  // t = ci * 9 + ky * 3 + kx
            sw3[l * C * 9 * CP + i] = co < C ? P.w3[l][(co * C + t / 9) * 9 + t % 9] : 0.0f;
        }
    for (int i = tid; i < C * CINP; i += TS_THREADS) {
        const int c = i / CINP, ci = i - c * CINP;
        sws[i] = (ci < P.stab_in) ? P.ws[c * P.stab_in + ci] : 0.0f;
    }
    for (int i = tid; i < C * CP; i += TS_THREADS) {
        const int c = i / CP, k = i - c * CP;
        swo[i] = k < C ? P.wo[c * C + k] : 0.0f;
    }
    for (int i = tid; i < 64; i += TS_THREADS) {
        const int t2 = i & 3, dv = (i >> 2) & 1, t1 = (i >> 3) & 3, du = i >> 5;
        skt[i] = P.kt[(1 - du) + 6 - 2 * t1][(1 - dv) + 6 - 2 * t2];
    }
    for (int i = tid; i < 56; i += TS_THREADS) skc[i] = (i & 7) < 7 ? P.kc[i >> 3][i & 7] : 0.0f;
    if (P.use_tma) {
        const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
        uint32_t done = 0;
        while (!done) {
            asm volatile(
                "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n selp.u32 %0, 1, 0, p;\n}\n"
                : "=r"(done)
                : "r"(bar_a)
                : "memory");
        }
        for (int i = tid; i < LW * LH; i += TS_THREADS) Lf[i] = (float)Lt[i];
    }
    __syncthreads();

    // ---- stage A on 2 x 2 quads of the region
    const int QW = RW / 2, nQ = (RH / 2) * QW;
    for (int q = tid; q < nQ; q += TS_THREADS) {
        const int qy = q / QW, qx = q - qy * QW;
        const int u0 = Y0 + 2 * qy, v0 = X0 + 2 * qx;  // even
        bool in[4];
        bool any_in = false;
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const int u = u0 + (p >> 1), v = v0 + (p & 1);
            in[p] = u >= 0 && u < H && v >= 0 && v < W;
            any_in |= in[p];
        }
        if (!any_in) continue;  // (filled by the fix-up pass)
        float x[4][CINP];
#pragma unroll
        for (int p = 0; p < 4; p++)
#pragma unroll
            for (int ci = 0; ci < CINP; ci++) x[p][ci] = 0.0f;
        {
            // channel 0: conv2d(latent, kron 7x7, zero padding) + latent (upsampling.py:189-196), sliding over the 8 rows
            // of the quad's 8 x 8 window; every output accumulates in (ka, kb) raster order
            const float *lp = Lf + (u0 - 3 - ly0) * LW + (v0 - 3 - lx0);
            float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f}, centre[4] = {0.0f, 0.0f, 0.0f, 0.0f};
            float wprev[7];
#pragma unroll
            for (int a = 0; a < 8; a++) {
                float r[8];
#pragma unroll
                for (int b = 0; b < 8; b++) r[b] = lp[a * LW + b];
                float wcur[7];
                if (a < 7) {
#pragma unroll
                    for (int b = 0; b < 7; b++) wcur[b] = skc[a * 8 + b];
                }
#pragma unroll
                for (int b = 0; b < 7; b++) {
                    if (a < 7) {  // row a is tap row ka = a of the outputs with dy = 0
                        acc[0] = __fmaf_rn(wcur[b], r[b], acc[0]);
                        acc[1] = __fmaf_rn(wcur[b], r[b + 1], acc[1]);
                    }
                    if (a >= 1) {  // and tap row ka = a - 1 of the outputs with dy = 1
                        acc[2] = __fmaf_rn(wprev[b], r[b], acc[2]);
                        acc[3] = __fmaf_rn(wprev[b], r[b + 1], acc[3]);
                    }
                }
                if (a == 3) { centre[0] = r[3]; centre[1] = r[4]; }
                if (a == 4) { centre[2] = r[3]; centre[3] = r[4]; }
                if (a < 7) {
#pragma unroll
                    for (int b = 0; b < 7; b++) wprev[b] = wcur[b];
                }
            }
#pragma unroll
            for (int p = 0; p < 4; p++) x[p][0] = __fadd_rn(acc[p], centre[p]);
        }
        {
            // channels 1 .. cc: transposed conv (8x8 kron, stride 2, replicate-padded input, crop 11; upsampling.py:312-325)
            const int qy0 = u0 >> 1, qx0 = v0 >> 1;  // (arithmetic shifts: u0, v0 may be negative on border tiles)
            int ro[5], co[5];
#pragma unroll
            for (int t = 0; t < 5; t++) {
                ro[t] = (clampi(qy0 - 2 + t, 0, ch - 1) - sy0) * SW;
                co[t] = clampi(qx0 - 2 + t, 0, cw - 1) - sx0;
            }
#pragma unroll
            for (int c = 0; c < CINP - 1; c++) {
                if (c < cc) {
                    const float *sp = St + c * SH * SW;
                    float win[5][5];
#pragma unroll
                    for (int i = 0; i < 5; i++)
#pragma unroll
                        for (int j = 0; j < 5; j++) win[i][j] = sp[ro[i] + co[j]];
#pragma unroll
                    for (int du = 0; du < 2; du++)
#pragma unroll
                        for (int dv = 0; dv < 2; dv++) {
                            float acc = 0.0f;
#pragma unroll
                            for (int t1 = 0; t1 < 4; t1++) {
                                const float4 w4 = *reinterpret_cast<const float4 *>(skt + ((du * 4 + t1) * 2 + dv) * 4);
                                acc = __fmaf_rn(w4.x, win[t1 + du][0 + dv], acc);
                                acc = __fmaf_rn(w4.y, win[t1 + du][1 + dv], acc);
                                acc = __fmaf_rn(w4.z, win[t1 + du][2 + dv], acc);
                                acc = __fmaf_rn(w4.w, win[t1 + du][3 + dv], acc);
                            }
                            x[du * 2 + dv][c + 1] = acc;
                        }
                }
            }
        }
        float o[4][C];
#pragma unroll
        for (int p = 0; p < 4; p++)
#pragma unroll
            for (int c = 0; c < C; c++) o[p][c] = sb1[c];
        for (int hh = 0; hh < hid; hh++) {
            float wv[CINP];
#pragma unroll
            for (int v = 0; v < CINP / 4; v++) {
                const float4 t = *reinterpret_cast<const float4 *>(sw0 + hh * CINP + 4 * v);
                wv[4 * v] = t.x; wv[4 * v + 1] = t.y; wv[4 * v + 2] = t.z; wv[4 * v + 3] = t.w;
            }
            float w1v[CP];
#pragma unroll
            for (int v = 0; v < CP / 4; v++) {
                const float4 t = *reinterpret_cast<const float4 *>(sw1 + hh * CP + 4 * v);
                w1v[4 * v] = t.x; w1v[4 * v + 1] = t.y; w1v[4 * v + 2] = t.z; w1v[4 * v + 3] = t.w;
            }
            const float bb = sb0[hh];
#pragma unroll
            for (int p = 0; p < 4; p++) {
                float a = bb;
#pragma unroll
                // (inputs and weights beyond cin are +0: fma(0, 0, a) == a bit for bit -- a starts from a bias that is never
                // -0 and a sum is -0 only if both terms are --, so no per-term test: a predicate copy per FMA was a third
                // of this loop's instructions)
                for (int ci = 0; ci < CINP; ci++) a = __fmaf_rn(wv[ci], x[p][ci], a);
                if (P.relu0) a = fmaxf(a, 0.0f);
#pragma unroll
                for (int c = 0; c < C; c++) o[p][c] = __fmaf_rn(w1v[c], a, o[p][c]);
            }
        }
#pragma unroll
        for (int p = 0; p < 4; p++) {
            if (!in[p]) continue;
            const int py = 2 * qy + (p >> 1), px = 2 * qx + (p & 1);
#pragma unroll
            for (int c = 0; c < C; c++) bufA[(c * RH + py) * RW + px] = P.relu1 ? fmaxf(o[p][c], 0.0f) : o[p][c];
            const int ty = py - n3e, tx = px - n3e;
            if (P.stab_in && ty >= 0 && ty < SF_TH && tx >= 0 && tx < SF_TW) {
#pragma unroll
                for (int c = 0; c < C; c++) {
                    float a = sbs[c];
#pragma unroll
                    for (int ci = 0; ci < CINP; ci++) a = __fmaf_rn(sws[c * CINP + ci], x[p][ci], a);  // (zero-padded: as above)
                    sstab[(c * SF_TH + ty) * SF_TW + tx] = a;
                }
            }
        }
    }
    __syncthreads();
    // ---- replicate padding on border tiles: out-of-frame positions of the region copy the clamped position
    if (Y0 < 0 || X0 < 0 || Y0 + RH > H || X0 + RW > W) {
        for (int pp = tid; pp < RH * RW; pp += TS_THREADS) {
            const int py = pp / RW, px = pp - py * RW;
            const int u = Y0 + py, v = X0 + px;
            if (u >= 0 && u < H && v >= 0 && v < W) continue;
            const int sy = clampi(u, 0, H - 1) - Y0, sx = clampi(v, 0, W - 1) - X0;
#pragma unroll
            for (int c = 0; c < C; c++) bufA[(c * RH + py) * RW + px] = bufA[(c * RH + sy) * RW + sx];
        }
        __syncthreads();
    }
    // ---- 3x3 layers: two horizontally adjacent outputs per thread
    const float *cur = bufA;
    int cwid = RW, chh = RH, off = n3e;
    for (int l = 0; l < n3 - 1; l++) {
        const int ow = cwid - 2, oh = chh - 2;
        const float *wl = sw3 + l * C * 9 * CP;
        for (int pp = tid; pp < (ow / 2) * oh; pp += TS_THREADS) {
            const int py = pp / (ow / 2), px = 2 * (pp - py * (ow / 2));
            const int gy = clampi(y0 - (off - 1) + py, 0, H - 1);
            const int by = gy - (y0 - off);
            const int bx0 = clampi(x0 - (off - 1) + px, 0, W - 1) - (x0 - off);
            const int bx1 = clampi(x0 - (off - 1) + px + 1, 0, W - 1) - (x0 - off);
            float acc0[C], acc1[C];
#pragma unroll
            for (int co = 0; co < C; co++) acc0[co] = acc1[co] = sb3[l * CP + co];
#pragma unroll
            for (int ci = 0; ci < C; ci++)
#pragma unroll
                for (int ky = 0; ky < 3; ky++) {
                    const float *row = cur + (ci * chh + by + ky - 1) * cwid;
                    float v0[3], v1[3];
                    if (bx1 == bx0 + 1) {
                        v0[0] = row[bx0 - 1]; v0[1] = row[bx0]; v0[2] = row[bx0 + 1];
                        v1[0] = v0[1]; v1[1] = v0[2]; v1[2] = row[bx0 + 2];
                    } else {
                        v0[0] = row[bx0 - 1]; v0[1] = row[bx0]; v0[2] = row[bx0 + 1];
                        v1[0] = row[bx1 - 1]; v1[1] = row[bx1]; v1[2] = row[bx1 + 1];
                    }
#pragma unroll
                    for (int kx = 0; kx < 3; kx++) {
                        float w[CP];
#pragma unroll
                        for (int v = 0; v < CP / 4; v++) {
                            const float4 t = *reinterpret_cast<const float4 *>(wl + ((ci * 3 + ky) * 3 + kx) * CP + 4 * v);
                            w[4 * v] = t.x; w[4 * v + 1] = t.y; w[4 * v + 2] = t.z; w[4 * v + 3] = t.w;
                        }
#pragma unroll
                        for (int co = 0; co < C; co++) {
                            acc0[co] = __fmaf_rn(w[co], v0[kx], acc0[co]);
                            acc1[co] = __fmaf_rn(w[co], v1[kx], acc1[co]);
                        }
                    }
                }
#pragma unroll
            for (int co = 0; co < C; co++) {
                float a0 = acc0[co], a1 = acc1[co];
                if (P.res3[l]) {
                    a0 = __fadd_rn(a0, cur[(co * chh + by) * cwid + bx0]);
                    a1 = __fadd_rn(a1, cur[(co * chh + by) * cwid + bx1]);
                }
                if (P.relu3[l]) { a0 = fmaxf(a0, 0.0f); a1 = fmaxf(a1, 0.0f); }
                bufB[(co * oh + py) * ow + px] = a0;
                bufB[(co * oh + py) * ow + px + 1] = a1;
            }
        }
        __syncthreads();
        cur = bufB;
        cwid = ow;
        chh = oh;
        off -= 1;
    }
    // ---- last stage on the tile (one pair of pixels per thread): last 3x3 layer (if any), + stabiliser, output
    // transform, frame tail, 64-bit stores
    const float M = P.M;
    float *uvq = sstab;  // 4:2:0 tail: rounded U, V of the tile where the stabiliser output was (own position, read first)
    for (int pp = tid; pp < (SF_TW / 2) * SF_TH; pp += TS_THREADS) {
        const int ty = pp / (SF_TW / 2), tx = 2 * (pp - ty * (SF_TW / 2));
        const int gy = y0 + ty, gx = x0 + tx;
        const bool in0 = gy < H && gx < W, in1 = gy < H && gx + 1 < W;
        const int tyc = in0 ? ty : 0, txc = in0 ? tx : 0;  // (out-of-frame pairs compute on a valid position, store nothing)
        const int by = tyc + off, bx0 = txc + off;
        const int bx1 = (in1 ? txc + 1 : txc) + off;
        float t0[C], t1[C];
        if (n3 > 0) {
            const int l = n3 - 1;
            const float *wl = sw3 + l * C * 9 * CP;
#pragma unroll
            for (int co = 0; co < C; co++) t0[co] = t1[co] = sb3[l * CP + co];
#pragma unroll
            for (int ci = 0; ci < C; ci++)
#pragma unroll
                for (int ky = 0; ky < 3; ky++) {
                    const float *row = cur + (ci * chh + by + ky - 1) * cwid;
                    float v0[3], v1[3];
                    v0[0] = row[bx0 - 1]; v0[1] = row[bx0]; v0[2] = row[bx0 + 1];
                    if (bx1 == bx0 + 1) {
                        v1[0] = v0[1]; v1[1] = v0[2]; v1[2] = row[bx0 + 2];
                    } else {
                        v1[0] = row[bx1 - 1]; v1[1] = row[bx1]; v1[2] = row[bx1 + 1];
                    }
#pragma unroll
                    for (int kx = 0; kx < 3; kx++) {
                        float w[CP];
#pragma unroll
                        for (int v = 0; v < CP / 4; v++) {
                            const float4 t = *reinterpret_cast<const float4 *>(wl + ((ci * 3 + ky) * 3 + kx) * CP + 4 * v);
                            w[4 * v] = t.x; w[4 * v + 1] = t.y; w[4 * v + 2] = t.z; w[4 * v + 3] = t.w;
                        }
#pragma unroll
                        for (int co = 0; co < C; co++) {
                            t0[co] = __fmaf_rn(w[co], v0[kx], t0[co]);
                            t1[co] = __fmaf_rn(w[co], v1[kx], t1[co]);
                        }
                    }
                }
#pragma unroll
            for (int co = 0; co < C; co++) {
                if (P.res3[l]) {
                    t0[co] = __fadd_rn(t0[co], cur[(co * chh + by) * cwid + bx0]);
                    t1[co] = __fadd_rn(t1[co], cur[(co * chh + by) * cwid + bx1]);
                }
                if (P.relu3[l]) { t0[co] = fmaxf(t0[co], 0.0f); t1[co] = fmaxf(t1[co], 0.0f); }
            }
        } else {
#pragma unroll
            for (int co = 0; co < C; co++) {
                t0[co] = cur[(co * chh + by) * cwid + bx0];
                t1[co] = cur[(co * chh + by) * cwid + bx1];
            }
        }
        if (P.stab_in) {
#pragma unroll
            for (int co = 0; co < C; co++) {
                t0[co] = __fadd_rn(t0[co], sstab[(co * SF_TH + tyc) * SF_TW + txc]);
                t1[co] = __fadd_rn(t1[co], sstab[(co * SF_TH + tyc) * SF_TW + (in1 ? txc + 1 : txc)]);
            }
        }
        float ov0[C], ov1[C];
#pragma unroll
        for (int co = 0; co < C; co++) {
            float a0 = sbo[co], a1 = sbo[co];
#pragma unroll
            for (int ci = 0; ci < C; ci++) {
                a0 = __fmaf_rn(swo[co * CP + ci], t0[ci], a0);
                a1 = __fmaf_rn(swo[co * CP + ci], t1[ci], a1);
            }
            ov0[co] = a0;
            ov1[co] = a1;
        }
        const size_t oi = (size_t)gy * W + gx;
        if (P.finish != 0) {
#pragma unroll
            for (int co = 0; co < C; co++) {
                ov0[co] = quant(ov0[co], M);
                ov1[co] = quant(ov1[co], M);
            }
        }
        const int n_full = P.finish == 2 ? 1 : C;  // planes stored at full resolution by this loop
#pragma unroll
        for (int co = 0; co < C; co++) {
            if (co < n_full) {
                float a0 = ov0[co], a1 = ov1[co];
                if (P.finish != 0) { a0 = quant(clamp01(a0), M); a1 = quant(clamp01(a1), M); }
                float *dst = P.out[co] + oi;
                if (in1 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) *reinterpret_cast<float2 *>(dst) = make_float2(a0, a1);
                else {
                    if (in0) P.out[co][oi] = a0;
                    if (in1) P.out[co][oi + 1] = a1;
                }
            }
        }
        if (P.finish == 2) {
            // (rounded U, V of own positions; read above, overwritten now)
            uvq[(0 * SF_TH + ty) * SF_TW + tx] = ov0[1 < C ? 1 : 0];
            uvq[(0 * SF_TH + ty) * SF_TW + tx + 1] = ov1[1 < C ? 1 : 0];
            uvq[(1 * SF_TH + ty) * SF_TW + tx] = ov0[2 < C ? 2 : 0];
            uvq[(1 * SF_TH + ty) * SF_TW + tx + 1] = ov1[2 < C ? 2 : 0];
        }
    }
    if (P.finish == 2) {
        __syncthreads();
        const int h2 = H / 2, w2 = W / 2;
        for (int pp = tid; pp < 2 * (SF_TW / 2) * (SF_TH / 2); pp += TS_THREADS) {
            const int c = pp / ((SF_TW / 2) * (SF_TH / 2)), r = pp - c * (SF_TW / 2) * (SF_TH / 2);
            const int by = r / (SF_TW / 2), bx = r - by * (SF_TW / 2);
            const int y2 = y0 / 2 + by, x2 = x0 / 2 + bx;
            if (y2 >= h2 || x2 >= w2) continue;
            const float *q = uvq + (c * SF_TH + 2 * by) * SF_TW + 2 * bx;
            float s = 0.0f;
            s = __fadd_rn(s, q[0]);
            s = __fadd_rn(s, q[1]);
            s = __fadd_rn(s, q[SF_TW]);
            s = __fadd_rn(s, q[SF_TW + 1]);
            P.out[1 + c][(size_t)y2 * w2 + x2] = quant(clamp01(__fdiv_rn(s, 4.0f)), M);
        }
    }
}

__global__ void k_add(float *__restrict__ a, const float *__restrict__ b, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = __fadd_rn(a[i], b[i]);
}

// legacy "nearest": src = min(floor(dst * (in/out as fp32)), in - 1)
__global__ void k_resize_nearest(const float *__restrict__ in, int h, int w, float *__restrict__ out, int H, int W,
                                 float sy, float sx) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int c = blockIdx.z;
    if (x >= W || y >= H) return;
    int yy = (int)floorf(__fmul_rn((float)y, sy));
    int xx = (int)floorf(__fmul_rn((float)x, sx));
    yy = yy > h - 1 ? h - 1 : yy;
    xx = xx > w - 1 ? w - 1 : xx;
    out[((size_t)c * H + y) * W + x] = in[((size_t)c * h + yy) * w + xx];
}

// F.interpolate(mode = bilinear | bicubic, align_corners=False, antialias=False), same operation order as
// oracle/ccoracle.c::resize_torch (PyTorch's separable CPU kernel): per axis src = fma(scale, dst + 0.5, -0.5),
// taps clamped to the grid, A = -0.75 cubic coefficients; value = sum_i wy[i] * (sum_j wx[j] * v[i][j]) as fma chains.
__device__ __forceinline__ float cubic_near(float x) {
    const float a = __fsub_rn(__fmul_rn(1.25f, x), 2.25f);
    return __fmaf_rn(__fmul_rn(a, x), x, 1.0f);
}
__device__ __forceinline__ float cubic_far(float x) {
    const float a = __fadd_rn(__fmul_rn(-0.75f, x), 3.75f);
    const float b = __fadd_rn(__fmul_rn(a, x), -6.0f);
    return __fadd_rn(__fmul_rn(b, x), 3.0f);
}
template <int MODE>  // 1 bilinear (2 taps), 2 bicubic (4 taps)
__device__ __forceinline__ void resize_taps(int n_in, int i, float scale, int (&idx)[4], float (&wt)[4]) {
    float src = __fmaf_rn(scale, __fadd_rn((float)i, 0.5f), -0.5f);
    if (MODE == 1 && src < 0.0f) src = 0.0f;
    int i0 = (int)floorf(src);
    if (i0 > n_in - 1) i0 = n_in - 1;
    float lam = __fsub_rn(src, (float)i0);
    lam = lam < 0.0f ? 0.0f : (lam > 1.0f ? 1.0f : lam);
    if (MODE == 1) {
        idx[0] = i0;
        idx[1] = i0 + (i0 < n_in - 1 ? 1 : 0);
        wt[0] = __fsub_rn(1.0f, lam);
        wt[1] = lam;
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) idx[j] = clampi(i0 + j - 1, 0, n_in - 1);
        const float x2 = __fsub_rn(1.0f, lam);
        wt[0] = cubic_far(__fadd_rn(lam, 1.0f));
        wt[1] = cubic_near(lam);
        wt[2] = cubic_near(x2);
        wt[3] = cubic_far(__fadd_rn(x2, 1.0f));
    }
}
template <int MODE>
__global__ void k_resize_torch(const float *__restrict__ in, int h, int w, float *__restrict__ out, int H, int W,
                               float sy, float sx) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int c = blockIdx.z;
    if (x >= W || y >= H) return;
    constexpr int N = MODE == 1 ? 2 : 4;
    int iy[4], ix[4];
    float wy[4], wx[4];
    resize_taps<MODE>(h, y, sy, iy, wy);
    resize_taps<MODE>(w, x, sx, ix, wx);
    const float *p = in + (size_t)c * h * w;
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < N; i++) {
        const float *row = p + (size_t)iy[i] * w;
        float r = __fmul_rn(wx[0], __ldg(row + ix[0]));
#pragma unroll
        for (int j = 1; j < N; j++) r = __fmaf_rn(wx[j], __ldg(row + ix[j]), r);
        acc = (i == 0) ? __fmul_rn(wy[0], r) : __fmaf_rn(wy[i], r, acc);
    }
    out[((size_t)c * H + y) * W + x] = acc;
}

// Common randomness (core/noise.py:18-55): sample k of the Park-Miller sequence, Box-Muller in f64.
// seed_j = a^j * seed_0 mod m is evaluated directly (square-and-multiply) instead of serially.
__device__ __forceinline__ uint64_t lcg_pow(uint64_t e) {
    const uint64_t m = 2147483647ULL;
    uint64_t r = 1, b = 16807ULL;
    while (e) {
        if (e & 1) r = (r * b) % m;
        b = (b * b) % m;
        e >>= 1;
    }
    return r;
}
__global__ void k_cr_noise(float *__restrict__ out, size_t first, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t m = 2147483647ULL;
    const size_t k = first + i;
    const uint64_t s1 = (lcg_pow(2 * k + 1) * 18101995ULL) % m;
    const uint64_t s2 = (s1 * 16807ULL) % m;
    const double u1 = (double)s1 / (double)m, u2 = (double)s2 / (double)m;
    // Box-Muller (noise.py:28-34) with the canonical log / cos of ccd_detmath.h: bit-identical to the oracle
    out[i] = (float)__dmul_rn(__dsqrt_rn(__dmul_rn(-2.0, ccdm_log(u1))), ccdm_cos(__dmul_rn(2 * 3.14159265359, u2)));
}

// Debug image of the canonical elementary functions (ccd_debug_detmath): y[i] = sin / cos / log (fn 0 / 1 / 2) of x[i]
__global__ void k_detmath(int fn, const double *__restrict__ x, double *__restrict__ y, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double v = x[i];
    y[i] = fn == 0 ? ccdm_sin(v) : (fn == 1 ? ccdm_cos(v) : ccdm_log(v));
}

__global__ void k_finish_444(const float *__restrict__ in, size_t n, float M, float *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = quant(clamp01(quant(in[i], M)), M);
}

__global__ void k_finish_420_uv(const float *__restrict__ in, int h, int w, float M, float *__restrict__ ou,
                                float *__restrict__ ov) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int c = blockIdx.z;  // 0: u, 1: v
    const int h2 = h / 2, w2 = w / 2;
    if (x >= w2 || y >= h2) return;
    const float *p = in + (size_t)(c + 1) * h * w;
    float s = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 2; dy++)
#pragma unroll
        for (int dx = 0; dx < 2; dx++) s = __fadd_rn(s, quant(p[(size_t)(2 * y + dy) * w + 2 * x + dx], M));
    float v = __fdiv_rn(s, 4.0f);
    (c == 0 ? ou : ov)[(size_t)y * w2 + x] = quant(clamp01(v), M);
}

inline dim3 grid2(int w, int h, int z = 1) { return dim3((w + 31) / 32, (h + 7) / 8, z); }
const dim3 kBlock2(32, 8, 1);

K1d make_k1d(const float *w1d, int k) {
    K1d r;
    for (int i = 0; i < 16; i++) r.w[i] = i < k ? w1d[i] : 0.0f;
    return r;
}

// kron(w, w) of a k-tap separable kernel: out[a * k + b] = w[a] * w[b]
void kron(const float *w, int k, float *out) {
    for (int a = 0; a < k; a++)
        for (int b = 0; b < k; b++) {
            volatile float p = w[a] * w[b];  // one rounded fp32 product, no contraction
            out[a * k + b] = p;
        }
}

}  // namespace

int ccd_ups_first(const int8_t *d_lat, int h, int w, float *d_out, cudaStream_t st) {
    size_t n = (size_t)h * w;
    k_ups_first<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_lat, n, d_out);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_ups_pre(const int8_t *d_lat, int h, int w, const float *w1d, int k, float *d_out, cudaStream_t st) {
    k_ups_pre<<<grid2(w, h), kBlock2, 0, st>>>(d_lat, h, w, make_k1d(w1d, k), k, d_out);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_ups_convt(const float *d_in, int c, int h, int w, const float *w1d, int k, float *d_out, int ht,
                  int wt, cudaStream_t st) {
    k_ups_convt<<<grid2(wt, ht, c), kBlock2, 0, st>>>(d_in, h, w, make_k1d(w1d, k), k, d_out, ht, wt);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_ups_level(const int8_t *d_lat, int th, int tw, const float *d_in, int cc, int ch, int cw, const float *wt1d,
                  const float *wc1d, float *d_out, cudaStream_t st) {
    UpsLevelParams P;
    P.lat = d_lat; P.in = d_in; P.out = d_out; P.cc = cc; P.ch = ch; P.cw = cw; P.th = th; P.tw = tw;
    kron(wt1d, 8, &P.kt[0][0]);
    kron(wc1d, 7, &P.kc[0][0]);
    k_ups_level<<<grid2(tw, th, cc + 1), kBlock2, 0, st>>>(P);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_syn_layer(const float *d_in, int h, int w, const SynLayerDev &L, float *d_out, cudaStream_t st) {
    k_syn_layer<<<grid2(w, h), kBlock2, 0, st>>>(d_in, h, w, L.cin, L.cout, L.k, L.residual, L.relu, L.w, L.b,
                                                 d_out);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_syn_pointwise2(const float *d_in, int h, int w, const SynLayerDev &L0, const SynLayerDev &L1,
                       float *d_out, cudaStream_t st) {
    // preconditions checked by the caller: k == 1, no residual, cin <= 16, cout(L1) <= 8
    size_t plane = (size_t)h * w;
    size_t smem = ((size_t)L0.cout * L0.cin + L0.cout + (size_t)L1.cout * L0.cout + L1.cout) * sizeof(float);
    k_syn_pw2<16, 8><<<(unsigned)((plane + 255) / 256), 256, smem, st>>>(
        d_in, plane, L0.cin, L0.cout, L1.cout, L0.relu, L1.relu, L0.w, L0.b, L1.w, L1.b, d_out);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

template <int CINP, int C>
static int launch_syn_fused(const SynFusedParams &P, cudaStream_t st) {
    constexpr int CP = (C + 3) & ~3;
    const int RW = SF_TW + 2 * P.n3, RH = SF_TH + 2 * P.n3;
    size_t fl = (size_t)P.hid * CINP + P.hid + (size_t)P.hid * CP + CP + 2 * C * C * 9 + 2 * CP + C * CINP + CP + C * CP + CP;
    fl += (size_t)C * RH * RW + (P.n3 == 2 ? (size_t)C * (RH - 2) * (RW - 2) : 0) + (size_t)C * SF_TH * SF_TW;
    const size_t smem = fl * sizeof(float);
    auto kern = k_syn_fused<CINP, C>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((P.w + SF_TW - 1) / SF_TW, (P.h + SF_TH - 1) / SF_TH, 1);
    kern<<<grid, SF_THREADS, smem, st>>>(P);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

bool ccd_syn_fused_family(int cin, const SynLayerDev *layers, int n_layers, const SynLayerDev *stab,
                          const SynLayerDev &ot) {
    if (n_layers < 2 || n_layers > 4) return false;
    const SynLayerDev &L0 = layers[0], &L1 = layers[1];
    const int C = L1.cout;
    if (L0.k != 1 || L1.k != 1 || L0.residual || L1.residual || cin > 16 || L0.cout > 256 || C < 2 || C > 5) return false;
    if (ot.cin != C || ot.cout != C) return false;
    for (int l = 2; l < n_layers; l++)
        if (layers[l].k != 3 || layers[l].cin != C || layers[l].cout != C) return false;
    return !stab || (stab->cin <= cin && stab->cout == C);
}

// returns -1 when the architecture is outside the fused family (caller falls back to the layer kernels)
int ccd_syn_fused(const float *d_in, int h, int w, int cin, const SynLayerDev *layers, int n_layers,
                  const SynLayerDev *stab, const SynLayerDev &ot, float *d_out, cudaStream_t st) {
    if (!ccd_syn_fused_family(cin, layers, n_layers, stab, ot)) return -1;
    const SynLayerDev &L0 = layers[0], &L1 = layers[1];
    const int C = L1.cout;
    SynFusedParams P;
    P.in = d_in; P.out = d_out; P.h = h; P.w = w; P.cin = cin; P.hid = L0.cout; P.n3 = n_layers - 2;
    P.relu0 = L0.relu; P.relu1 = L1.relu;
    for (int l = 0; l < 2; l++) {
        const bool on = l < P.n3;
        P.res3[l] = on ? layers[2 + l].residual : 0;
        P.relu3[l] = on ? layers[2 + l].relu : 0;
        P.w3[l] = on ? layers[2 + l].w : nullptr;
        P.b3[l] = on ? layers[2 + l].b : nullptr;
    }
    P.stab_in = stab ? stab->cin : 0;
    P.w0 = L0.w; P.b0 = L0.b; P.w1 = L1.w; P.b1 = L1.b;
    P.ws = stab ? stab->w : nullptr; P.bs = stab ? stab->b : nullptr;
    P.wo = ot.w; P.bo = ot.b;
    const int cinp = cin <= 4 ? 4 : (cin <= 8 ? 8 : 16);
#define SF_CASE(CI, CC) if (cinp == CI && C == CC) return launch_syn_fused<CI, CC>(P, st)
    SF_CASE(4, 2); SF_CASE(4, 3); SF_CASE(4, 4); SF_CASE(4, 5);
    SF_CASE(8, 2); SF_CASE(8, 3); SF_CASE(8, 4); SF_CASE(8, 5);
    SF_CASE(16, 2); SF_CASE(16, 3); SF_CASE(16, 4); SF_CASE(16, 5);
#undef SF_CASE
    return -1;
}

// ---- batched float tail: host side -----------------------------------------------------------------------
size_t ccd_tail_job_bytes(void) { return sizeof(TailSynJob); }
size_t ccd_tail_level_job_bytes(void) { return sizeof(UpsLevelJob); }

void ccd_tail_fill_level(void *dst, const int8_t *lat, const float *in, const int8_t *in8, float *out, int cc, int ch,
                         int cw, int th, int tw, const float *wt1d, const float *wc1d) {
    UpsLevelJob J;
    memset(&J, 0, sizeof(J));
    J.lat = lat; J.in = in; J.in8 = in8; J.out = out; J.cc = cc; J.ch = ch; J.cw = cw; J.th = th; J.tw = tw;
    kron(wt1d, 8, &J.kt[0][0]);
    kron(wc1d, 7, &J.kc[0][0]);
    memcpy(dst, &J, sizeof(J));
}

int ccd_tail_launch_level(const void *d_jobs, int n_jobs, int planes, int max_tw, int max_th, cudaStream_t st) {
    const dim3 grid((max_tw + 31) / 32, (max_th + 7) / 8, (unsigned)(n_jobs * planes));
    k_ups_level_b<<<grid, kBlock2, 0, st>>>(reinterpret_cast<const UpsLevelJob *>(d_jobs), planes);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

namespace {
typedef int (*PFN_encodeTiled)(void *tensorMap, int dataType, unsigned rank, void *globalAddress, const uint64_t *globalDim,
                               const uint64_t *globalStrides, const uint32_t *boxDim, const uint32_t *elementStrides,
                               int interleave, int swizzle, int l2Promotion, int oobFill);
PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
        cudaGetLastError();
    }
    return fn;
}
}  // namespace

// Fills one TailSynJob (host memory).  The tiles are staged with TMA unless the pitches / addresses are ones that
// cuTensorMapEncodeTiled does not take (plain loads then).
void ccd_tail_fill_syn(void *dst, const CcdTailSynDesc &T) {
    const int n_layers = T.n_layers;
    const SynLayerDev &L0 = T.layers[0], &L1 = T.layers[1];
    TailSynJob J;
    memset(&J, 0, sizeof(J));
    J.lat = T.lat; J.stk = T.stk; J.stk8 = T.stk8;
    for (int c = 0; c < 5; c++) J.out[c] = T.out[c];
    J.h = T.h; J.w = T.w; J.ch = T.ch; J.cw = T.cw; J.cin = T.cin; J.hid = L0.cout; J.n3 = n_layers - 2;
    J.relu0 = L0.relu; J.relu1 = L1.relu;
    for (int l = 0; l < 2; l++) {
        const bool on = l < J.n3;
        J.res3[l] = on ? T.layers[2 + l].residual : 0;
        J.relu3[l] = on ? T.layers[2 + l].relu : 0;
        J.w3[l] = on ? T.layers[2 + l].w : nullptr;
        J.b3[l] = on ? T.layers[2 + l].b : nullptr;
    }
    J.stab_in = T.stab ? T.stab->cin : 0;
    J.w0 = L0.w; J.b0 = L0.b; J.w1 = L1.w; J.b1 = L1.b;
    J.ws = T.stab ? T.stab->w : nullptr; J.bs = T.stab ? T.stab->b : nullptr;
    J.wo = T.ot.w; J.bo = T.ot.b;
    J.finish = T.finish;
    J.M = T.M;
    kron(T.wt1d, 8, &J.kt[0][0]);
    kron(T.wc1d, 7, &J.kc[0][0]);
    // TMA descriptors (CU_TENSOR_MAP_DATA_TYPE_UINT8 = 0, FLOAT32 = 7; no interleave, no swizzle, L2 promotion 128 B,
    // out-of-bounds elements read as zero)
    J.use_tma = 0;
    PFN_encodeTiled enc = get_encode_tiled();
    const int cc = T.cin - 1;
    if (enc && T.allow_tma && !T.stk8 && (T.w % 16) == 0 && (T.cw % 4) == 0 && (reinterpret_cast<uintptr_t>(T.lat) % 16) == 0 &&
        (reinterpret_cast<uintptr_t>(T.stk) % 16) == 0) {
        const uint64_t gd0[2] = {(uint64_t)T.w, (uint64_t)T.h};
        const uint64_t gs0[1] = {(uint64_t)T.w};
        const int n3t = ts_n3e(J.n3);  // halo of the staged tiles
        const uint32_t bx0[2] = {(uint32_t)ts_lw(n3t), (uint32_t)ts_lh(n3t)};
        const uint32_t es[3] = {1, 1, 1};
        const uint64_t gd1[3] = {(uint64_t)T.cw, (uint64_t)T.ch, (uint64_t)cc};
        const uint64_t gs1[2] = {(uint64_t)T.cw * 4, (uint64_t)T.cw * 4 * (uint64_t)T.ch};
        const uint32_t bx1[3] = {(uint32_t)ts_sw(n3t), (uint32_t)ts_sh(n3t), (uint32_t)cc};
        const int r0 = enc(J.tmap_lat, 0, 2, const_cast<int8_t *>(T.lat), gd0, gs0, bx0, es, 0, 0, 1, 0);
        const int r1 = enc(J.tmap_stk, 7, 3, const_cast<float *>(T.stk), gd1, gs1, bx1, es, 0, 0, 1, 0);
        J.use_tma = (r0 == 0 && r1 == 0) ? 1 : 0;
    }
    memcpy(dst, &J, sizeof(J));
}

template <int CINP, int C>
static int launch_tail_syn(const void *d_jobs, int n_jobs, int n3_max, int hid_max, int max_w, int max_h, cudaStream_t st) {
    constexpr int CP = (C + 3) & ~3;
    const int n3t = ts_n3e(n3_max);
    const int RW = SF_TW + 2 * n3t, RH = SF_TH + 2 * n3t;
    size_t bytes = 128 + (((size_t)ts_lw(n3t) * ts_lh(n3t) + 127) & ~(size_t)127);
    size_t fl = (((size_t)(CINP - 1) * ts_sh(n3t) * ts_sw(n3t) + 31) & ~(size_t)31);
    fl += (size_t)ts_lw(n3t) * ts_lh(n3t);
    fl += (size_t)hid_max * CINP + ((hid_max + 3) & ~3) + (size_t)hid_max * CP + CP + 2 * C * 9 * CP + 2 * CP + C * CINP + CP + C * CP + CP + 64 + 56;
    fl += (size_t)C * RH * RW + (n3_max == 2 ? (size_t)C * (RH - 2) * (RW - 2) : 0) + (size_t)C * SF_TH * SF_TW;
    const size_t smem = bytes + fl * sizeof(float);
    auto kern = k_tail_syn<CINP, C>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((max_w + SF_TW - 1) / SF_TW, (max_h + SF_TH - 1) / SF_TH, (unsigned)n_jobs);
    kern<<<grid, TS_THREADS, smem, st>>>(reinterpret_cast<const TailSynJob *>(d_jobs));
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

// all jobs of one launch share (cinp, C); n3 / hid / sizes may differ (shared memory sized for the maxima)
int ccd_tail_launch_syn(const void *d_jobs, int n_jobs, int cinp, int C, int n3_max, int hid_max, int max_w, int max_h,
                        cudaStream_t st) {
#define TS_CASE(CI, CC) if (cinp == CI && C == CC) return launch_tail_syn<CI, CC>(d_jobs, n_jobs, n3_max, hid_max, max_w, max_h, st)
    TS_CASE(4, 2); TS_CASE(4, 3); TS_CASE(4, 4); TS_CASE(4, 5);
    TS_CASE(8, 2); TS_CASE(8, 3); TS_CASE(8, 4); TS_CASE(8, 5);
    TS_CASE(16, 2); TS_CASE(16, 3); TS_CASE(16, 4); TS_CASE(16, 5);
#undef TS_CASE
    return -1;
}

int ccd_syn_add(float *d_a, const float *d_b, size_t n, cudaStream_t st) {
    k_add<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_a, d_b, n);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_resize_nearest(const float *d_in, int c, int h, int w, float *d_out, int H, int W, cudaStream_t st) {
    k_resize_nearest<<<grid2(W, H, c), kBlock2, 0, st>>>(d_in, h, w, d_out, H, W, (float)h / (float)H,
                                                         (float)w / (float)W);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_resize_torch(const float *d_in, int c, int h, int w, float *d_out, int H, int W, int mode, float sy, float sx,
                     cudaStream_t st) {
    if (mode == 1)
        k_resize_torch<1><<<grid2(W, H, c), kBlock2, 0, st>>>(d_in, h, w, d_out, H, W, sy, sx);
    else
        k_resize_torch<2><<<grid2(W, H, c), kBlock2, 0, st>>>(d_in, h, w, d_out, H, W, sy, sx);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_cr_noise(float *d_out, size_t first, size_t n, cudaStream_t st) {
    k_cr_noise<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_out, first, n);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_detmath(int fn, const double *d_x, double *d_y, size_t n, cudaStream_t st) {
    k_detmath<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(fn, d_x, d_y, n);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

// ---- output packing (io/format/yuv.py:150-162, ppm.py:160-203): finished planes -> integer samples.
// Planar: thread = 4 consecutive samples of one plane (one float4 load, one 4- or 8-byte store).
template <typename T>
__global__ void k_pack_planar(const float *__restrict__ p0, const float *__restrict__ p1, const float *__restrict__ p2,
                              size_t n0, size_t n1, float M, T *__restrict__ out) {
    const size_t total4 = (n0 + 3) / 4 + 2 * ((n1 + 3) / 4);
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < total4; q += (size_t)gridDim.x * blockDim.x) {
        const size_t q0 = (n0 + 3) / 4, q1 = (n1 + 3) / 4;
        const float *src;
        size_t base, n, off;
        if (q < q0) { src = p0; base = 0; n = n0; off = q * 4; }
        else if (q < q0 + q1) { src = p1; base = n0; n = n1; off = (q - q0) * 4; }
        else { src = p2; base = n0 + n1; n = n1; off = (q - q0 - q1) * 4; }
        T v[4];
        if (off + 4 <= n && ((reinterpret_cast<uintptr_t>(src + off) & 15) == 0)) {
            const float4 f = __ldg(reinterpret_cast<const float4 *>(src + off));
            v[0] = (T)rintf(__fmul_rn(f.x, M)); v[1] = (T)rintf(__fmul_rn(f.y, M));
            v[2] = (T)rintf(__fmul_rn(f.z, M)); v[3] = (T)rintf(__fmul_rn(f.w, M));
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = (off + k < n) ? (T)rintf(__fmul_rn(__ldg(src + off + k), M)) : (T)0;
        }
        T *dst = out + base + off;
        if (off + 4 <= n && ((reinterpret_cast<uintptr_t>(dst) & (4 * sizeof(T) - 1)) == 0)) {
            if (sizeof(T) == 1) *reinterpret_cast<uchar4 *>(dst) = make_uchar4(v[0], v[1], v[2], v[3]);
            else *reinterpret_cast<ushort4 *>(dst) = make_ushort4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (off + k < n) dst[k] = v[k];
        }
    }
}
// Interleaved [H][W][3]: thread = 4 pixels = 12 samples (three float4 loads, 12 or 24 contiguous bytes out).
template <typename T>
__global__ void k_pack_hwc(const float *__restrict__ p0, const float *__restrict__ p1, const float *__restrict__ p2, size_t n,
                           float M, T *__restrict__ out) {
    const size_t nq = (n + 3) / 4;
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (size_t)gridDim.x * blockDim.x) {
        const size_t off = q * 4;
        T v[12];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const size_t i = off + k < n ? off + k : n - 1;
            v[3 * k] = (T)rintf(__fmul_rn(__ldg(p0 + i), M));
            v[3 * k + 1] = (T)rintf(__fmul_rn(__ldg(p1 + i), M));
            v[3 * k + 2] = (T)rintf(__fmul_rn(__ldg(p2 + i), M));
        }
        T *dst = out + off * 3;
        if (off + 4 <= n) {
            if (sizeof(T) == 1) {
                uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);  // off * 3 is a multiple of 12: 4-byte aligned
#pragma unroll
                for (int k = 0; k < 3; k++)
                    d32[k] = (uint32_t)v[4 * k] | ((uint32_t)v[4 * k + 1] << 8) | ((uint32_t)v[4 * k + 2] << 16) |
                             ((uint32_t)v[4 * k + 3] << 24);
            } else {
                uint2 *d64 = reinterpret_cast<uint2 *>(dst);        // 24 bytes: 8-byte aligned
#pragma unroll
                for (int k = 0; k < 3; k++)
                    d64[k] = make_uint2((uint32_t)v[4 * k] | ((uint32_t)v[4 * k + 1] << 16),
                                        (uint32_t)v[4 * k + 2] | ((uint32_t)v[4 * k + 3] << 16));
            }
        } else {
            for (int k = 0; k < 12; k++)
                if (off * 3 + k < n * 3) dst[k] = v[k];
        }
    }
}

int ccd_pack(const float *const planes[3], int h, int w, int cs, int bitdepth, int sample_bytes, int interleaved,
             void *d_out, cudaStream_t st) {
    const float M = (float)((1 << bitdepth) - 1);
    const size_t n0 = (size_t)h * w, n1 = (size_t)(h >> cs) * (w >> cs);
    const unsigned blocks = 132 * 8;  // grid-stride loop: 8 CTAs per SM of an H100
    if (interleaved) {
        if (sample_bytes == 1) k_pack_hwc<uint8_t><<<blocks, 256, 0, st>>>(planes[0], planes[1], planes[2], n0, M, (uint8_t *)d_out);
        else k_pack_hwc<uint16_t><<<blocks, 256, 0, st>>>(planes[0], planes[1], planes[2], n0, M, (uint16_t *)d_out);
    } else {
        if (sample_bytes == 1) k_pack_planar<uint8_t><<<blocks, 256, 0, st>>>(planes[0], planes[1], planes[2], n0, n1, M, (uint8_t *)d_out);
        else k_pack_planar<uint16_t><<<blocks, 256, 0, st>>>(planes[0], planes[1], planes[2], n0, n1, M, (uint16_t *)d_out);
    }
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

// n samples that already lie in output order (the planes of a batch of finished frames, one after the other)
int ccd_pack_flat(const float *d_in, size_t n, int bitdepth, int sample_bytes, void *d_out, cudaStream_t st) {
    const float M = (float)((1 << bitdepth) - 1);
    const unsigned blocks = 132 * 8;  // grid-stride loop: 8 CTAs per SM of an H100
    if (sample_bytes == 1) k_pack_planar<uint8_t><<<blocks, 256, 0, st>>>(d_in, d_in, d_in, n, 0, M, (uint8_t *)d_out);
    else k_pack_planar<uint16_t><<<blocks, 256, 0, st>>>(d_in, d_in, d_in, n, 0, M, (uint16_t *)d_out);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

// ---- distortion against the source, the mirror image of the packing above: each decoded sample goes back to its
// integer kd = rint(x * M) and is compared with the source sample ks as it was uploaded (uint8 / uint16, planar or
// [H][W][3], never widened on the host).  A thread owns pixels of the luma grid; with 4:2:0 chroma only the thread of
// the even (x, y) counts the chroma sample, the others read it only for the error map.  Sums are integers: exact, and
// the same whatever the order of the atomics.
// Sample s of plane c of a frame pair whose planes hold n0 and n1 samples (computed once per kernel): the decoded sample,
// the source integer ks and the planar (FrameData) index that bad_index reports.  The caller tests CCD_OFF_GRID(d)
// under its own condition.
struct SamplePair { DecodedSample d; int ks; unsigned pidx; };
static __device__ __forceinline__ SamplePair read_pair(const FramePairDev &F, int c, unsigned s, unsigned n0, unsigned n1) {
    const DecodedSample D = read_decoded(F.p[c], s, F.M);
    const unsigned pidx = c == 0 ? s : n0 + (unsigned)(c - 1) * n1 + s;
    return SamplePair{D, source_sample(F.src, F.wide, F.hwc ? (size_t)s * 3 + c : (size_t)pidx), pidx};
}

__global__ void __launch_bounds__(256) k_frame_dist(const DistJobDev *__restrict__ jobs) {
    const DistJobDev &J = jobs[blockIdx.y];
    const unsigned w = (unsigned)J.w, cs = (unsigned)J.cs, n0 = (unsigned)J.h * w;
    const unsigned wc = w >> cs, n1 = ((unsigned)J.h >> cs) * wc;
    const bool want_map = J.map != nullptr;
    unsigned long long s[3] = {0ull, 0ull, 0ull}, bad = ~0ull;
    unsigned mx[3] = {0u, 0u, 0u};
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n0; i += gridDim.x * blockDim.x) {
        const unsigned y = i / w, x = i - y * w;
        const bool own = ((x | y) & cs) == 0;  // counts the chroma sample (always, without subsampling)
        unsigned long long e = 0ull;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            if (c > 0 && !own && !want_map) continue;
            const SamplePair P = read_pair(J, c, c == 0 ? i : (y >> cs) * wc + (x >> cs), n0, n1);
            const unsigned a = (unsigned)abs((int)P.d.kd - P.ks);
            const unsigned long long d2 = (unsigned long long)a * a;
            e += d2;
            if (c == 0 || own) {
                s[c] += d2;
                mx[c] = max(mx[c], a);
                if (CCD_OFF_GRID(P.d)) bad = min(bad, (unsigned long long)P.pidx);
            }
        }
        if (want_map) J.map[i] = __fdiv_rn(__ull2float_rn(e), J.M2);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        for (int o = 16; o > 0; o >>= 1) s[c] += __shfl_down_sync(0xffffffffu, s[c], o);
        mx[c] = __reduce_max_sync(0xffffffffu, mx[c]);
    }
    for (int o = 16; o > 0; o >>= 1) bad = min(bad, __shfl_down_sync(0xffffffffu, bad, o));
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            if (s[c]) atomicAdd(J.sse + c, s[c]);
            if (mx[c]) atomicMax(J.max_abs + c, mx[c]);
        }
        if (bad != ~0ull) atomicMin(J.bad, bad);
    }
}

int ccd_dist_launch(const DistJobDev *d_jobs, int n_jobs, int64_t max_pixels, int n_sm, cudaStream_t st) {
    // about 16 CTAs per SM over the whole call, at least one per job
    const int64_t want = (max_pixels + 255) / 256, cap = ((int64_t)n_sm * 16 + n_jobs - 1) / n_jobs;
    const int64_t per_job = want < cap ? want : cap;
    k_frame_dist<<<dim3((unsigned)per_job, (unsigned)n_jobs, 1), 256, 0, st>>>(d_jobs);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

// ---- Tiled local statistics against the source: MS-SSIM (DESIGN §4.6) and VIF (§4.12), one scale per launch.  A CTA
// of kTileWarps warps takes one CCD_SSIM_T x CCD_SSIM_T tile of one plane at one scale, stages it with its halo, forms
// the five local moments x, y, x^2, y^2, x y with a separable window, and reduces two per-pixel terms to one f64
// partial each, in a fixed order.
namespace {
constexpr int kTileWarps = 8;
constexpr int kTileK = 4;  // consecutive outputs per thread in either moment pass
static_assert(CCD_SSIM_T == 32 && CCD_SSIM_T / kTileK == kTileWarps, "vertical pass: lane = column, warp = K rows");
static_assert((CCD_SSIM_T / 2) * (CCD_SSIM_T / 2) == 32 * kTileWarps, "one next-level sample per thread");
}  // namespace

static __device__ __forceinline__ void report_bad(unsigned long long bad, unsigned long long *out, int tid) {
    for (int o = 16; o > 0; o >>= 1) bad = min(bad, __shfl_down_sync(0xffffffffu, bad, o));
    if ((tid & 31) == 0 && bad != ~0ull) atomicMin(out, bad);
}

// The plane c and tile t of this CTA (MS-SSIM, VIF, PSNR-HVS-M: blockIdx.x = tile over the job's planes, plane 0's
// tiles first), and that plane's h x w at this scale.  side(n): a side of n samples at this scale; tiles(h, w): the
// tiles of a plane.  The host's TilePlan (ccd_api.cu) lays out the call from the same two.
struct PlaneTile { int c, t, h, w; };  // c == 3: past the job's last tile
template <class Side, class Tiles>
static __device__ __forceinline__ PlaneTile locate_tile(const FramePairDev &F, Side side, Tiles tiles) {
    int c = 0, t = (int)blockIdx.x, h = 0, w = 0;
    for (;; c++) {
        if (c == 3) break;
        h = side(c ? F.h >> F.cs : F.h);
        w = side(c ? F.w >> F.cs : F.w);
        const int n = tiles(h, w);
        if (t < n) break;
        t -= n;
    }
    return PlaneTile{c, t, h, w};
}

// Horizontal pass: rows [0, In) of the staged [In][In] images sx, sy, filtered with the NT taps g at T positions per
// row, into sh[5][In][T].  A thread takes K consecutive outputs of one row at a time.
template <int NT, int In, class S>
static __device__ __forceinline__ void moments_h(const S *sx, const S *sy, const double *g, double *sh, int tid) {
    constexpr int T = CCD_SSIM_T, K = kTileK;
    for (int task = tid; task < In * (T / K); task += 32 * kTileWarps) {
        const int r = task / (T / K), q0 = task % (T / K) * K;
        const S *rx = sx + r * In + q0, *ry = sy + r * In + q0;
        double m[5][K];
#pragma unroll
        for (int k = 0; k < K; k++)
#pragma unroll
            for (int e = 0; e < 5; e++) m[e][k] = 0.0;
#pragma unroll
        for (int i = 0; i < K + NT - 1; i++) {
            const double x = rx[i], y = ry[i], v[5] = {x, y, x * x, y * y, x * y};
#pragma unroll
            for (int k = 0; k < K; k++) {
                if (i - k < 0 || i - k > NT - 1) continue;
#pragma unroll
                for (int e = 0; e < 5; e++) m[e][k] = fma(g[i - k], v[e], m[e][k]);
            }
        }
#pragma unroll
        for (int e = 0; e < 5; e++)
#pragma unroll
            for (int k = 0; k < K; k++) sh[(e * In + r) * T + q0 + k] = m[e][k];
    }
}

// Vertical pass: the five moments of column q at rows r0 .. r0 + K - 1, from sh[5][In][T].
template <int NT, int In>
static __device__ __forceinline__ void moments_v(const double *sh, const double *g, int q, int r0, double (&m)[5][kTileK]) {
    constexpr int T = CCD_SSIM_T, K = kTileK;
#pragma unroll
    for (int k = 0; k < K; k++)
#pragma unroll
        for (int e = 0; e < 5; e++) m[e][k] = 0.0;
#pragma unroll
    for (int i = 0; i < K + NT - 1; i++) {
#pragma unroll
        for (int e = 0; e < 5; e++) {
            const double v = sh[(e * In + r0 + i) * T + q];
#pragma unroll
            for (int k = 0; k < K; k++)
                if (i - k >= 0 && i - k <= NT - 1) m[e][k] = fma(g[i - k], v, m[e][k]);
        }
    }
}

// The CTA's two sums a, b, handed to thread 0's store(a, b): a lane butterfly, then the warps in order (sred: [warps][2])
template <class Store>
static __device__ __forceinline__ void tile_sums(double &a, double &b, double *sred, int tid, Store store) {
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((tid & 31) == 0) {
        sred[2 * (tid >> 5)] = a;
        sred[2 * (tid >> 5) + 1] = b;
    }
    __syncthreads();
    if (tid == 0) {
        double pa = 0.0, pb = 0.0;
        for (int wi = 0; wi < kTileWarps; wi++) {
            pa += sred[2 * wi];
            pb += sred[2 * wi + 1];
        }
        store(pa, pb);
    }
}

// ---- MS-SSIM.  x = the decoded image, y = the source, both as the integer sums S_j of the 4^j samples a level-j
// sample covers: below 65535 * 256 < 2^24, so staged exactly in fp32 (68 KB of shared memory: three CTAs per SM);
// every moment is formed in f64 on S_j and scaled by 4^-j or 16^-j afterwards, which is exact.  Per tile: stage
// (T + 10)^2 samples of both images, write the next level's T/2 x T/2 samples, filter the five moments horizontally
// then vertically (11 taps, valid positions only), and add cs and l * cs of the tile's valid positions in a fixed
// order into one f64 partial each.
namespace {
constexpr int kSsimIn = CCD_SSIM_T + CCD_SSIM_HALO;  // staged rows and columns
constexpr size_t kSsimSmem = sizeof(float) * 2 * kSsimIn * kSsimIn + sizeof(double) * (5 * kSsimIn * CCD_SSIM_T + 2 * kTileWarps);
struct SsimArgs {
    double g[11];
    int scale;
};
}  // namespace

__global__ void __launch_bounds__(32 * kTileWarps, 3) k_frame_ssim(const SsimJobDev *__restrict__ jobs, const SsimArgs a) {
    constexpr int T = CCD_SSIM_T, K = kTileK;
    extern __shared__ double ssim_sm[];
    double *sh = ssim_sm;                                 // [5][kSsimIn][T]: the horizontal pass
    float *sx = reinterpret_cast<float *>(sh + 5 * kSsimIn * T), *sy = sx + kSsimIn * kSsimIn;  // [kSsimIn][kSsimIn]
    double *sred = reinterpret_cast<double *>(sy + kSsimIn * kSsimIn);  // [warps][2]
    const SsimJobDev &J = jobs[blockIdx.y];
    const int j = a.scale, tid = (int)threadIdx.x;
    const auto [c, t, h, w] = locate_tile(J, [j](int n) { return n >> j; }, ccd_ssim_tiles);
    if (c == 3) return;
    const int tw = (w + T - 1) / T, y0 = t / tw * T, x0 = t % tw * T;

    unsigned long long bad = ~0ull;
    const unsigned n0 = (unsigned)J.h * J.w, n1 = (unsigned)(J.h >> J.cs) * (unsigned)(J.w >> J.cs);
    for (int i = tid; i < kSsimIn * kSsimIn; i += 32 * kTileWarps) {
        const int r = i / kSsimIn, q = i - r * kSsimIn, y = y0 + r, x = x0 + q;
        float vx = 0.0f, vy = 0.0f;  // integers below 2^24: exact
        if (y < h && x < w) {
            const unsigned s = (unsigned)y * (unsigned)w + (unsigned)x;
            if (j == 0) {
                const SamplePair P = read_pair(J, c, s, n0, n1);
                vx = P.d.kd;
                vy = (float)P.ks;
                if (r < T && q < T && CCD_OFF_GRID(P.d)) bad = min(bad, (unsigned long long)P.pidx);
            } else {
                const uint2 v = J.lvl[c][j][s];
                vx = (float)v.x;
                vy = (float)v.y;
            }
        }
        sx[i] = vx;
        sy[i] = vy;
    }
    if (j == 0) report_bad(bad, J.bad, tid);
    __syncthreads();

    if (j + 1 < CCD_SSIM_SCALES) {  // the next level: floor sizes, an odd last row or column is dropped
        const int r = tid / (T / 2), q = tid % (T / 2), Y = (y0 >> 1) + r, X = (x0 >> 1) + q;
        if (Y < (h >> 1) && X < (w >> 1)) {
            const int k = 2 * r * kSsimIn + 2 * q;
            J.lvl[c][j + 1][(size_t)Y * (w >> 1) + X] =
                make_uint2((unsigned)(sx[k] + sx[k + 1] + sx[k + kSsimIn] + sx[k + kSsimIn + 1]),
                           (unsigned)(sy[k] + sy[k + 1] + sy[k + kSsimIn] + sy[k + kSsimIn + 1]));
        }
    }

    // the f64 products of the horizontal pass are exact: S_j < 2^24
    moments_h<11, kSsimIn>(sx, sy, a.g, sh, tid);
    __syncthreads();

    double s_cs = 0.0, s_ssim = 0.0;
    {
        const int q = tid & 31, r0 = (tid >> 5) * K;
        double m[5][K];
        moments_v<11, kSsimIn>(sh, a.g, q, r0, m);
        const double s1 = ldexp(1.0, -2 * j), s2 = __dmul_rn(s1, s1);
        const int x = x0 + q, wo = w - CCD_SSIM_HALO, ho = h - CCD_SSIM_HALO;
#pragma unroll
        for (int k = 0; k < K; k++) {
            const int y = y0 + r0 + k;
            if (x >= wo || y >= ho) continue;
            // no contraction: identical images give cs = l = 1 exactly
            const double mx = __dmul_rn(m[0][k], s1), my = __dmul_rn(m[1][k], s1);
            const double mxx = __dmul_rn(mx, mx), myy = __dmul_rn(my, my), mxy = __dmul_rn(mx, my);
            const double vx = __dsub_rn(__dmul_rn(m[2][k], s2), mxx), vy = __dsub_rn(__dmul_rn(m[3][k], s2), myy);
            const double cxy = __dsub_rn(__dmul_rn(m[4][k], s2), mxy);
            const double cs = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, cxy), J.C2), __dadd_rn(__dadd_rn(vx, vy), J.C2));
            const double l = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, mxy), J.C1), __dadd_rn(__dadd_rn(mxx, myy), J.C1));
            const double ls = __dmul_rn(l, cs);
            s_cs = __dadd_rn(s_cs, cs);
            s_ssim = __dadd_rn(s_ssim, ls);
            if (j == 0 && J.map[c]) J.map[c][(size_t)y * wo + x] = __double2float_rn(ls);
        }
    }
    tile_sums(s_cs, s_ssim, sred, tid, [&](double pc, double ps) {
        J.part[j][2 * blockIdx.x] = pc;
        J.part[j][2 * blockIdx.x + 1] = ps;
    });
}

int ccd_ssim_launch(const SsimJobDev *d_jobs, int n_jobs, const int max_tiles[CCD_SSIM_SCALES], const double g[11],
                    cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_frame_ssim, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSsimSmem);
    if (e != cudaSuccess) return (int)e;
    SsimArgs a;
    memcpy(a.g, g, sizeof(a.g));
    for (int j = 0; j < CCD_SSIM_SCALES; j++) {  // scale j + 1 reads the level scale j wrote: stream order
        a.scale = j;
        k_frame_ssim<<<dim3((unsigned)max_tiles[j], (unsigned)n_jobs, 1), 32 * kTileWarps, kSsimSmem, st>>>(d_jobs, a);
        g_ccd_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    }
    return 0;
}

// ---- VIF.  x = the decoded image (distorted), y = the source (reference), both in 8-bit units and f64 from the start:
// v = k * 255 / M at scale 0, the filtered and decimated values at scales 1..3.  Per tile of scale S: stage
// (T + N_S - 1)^2 samples of both images (61 to 98 KB of shared memory: at least two CTAs per SM), write the next scale's
// T/2 x T/2 samples (N_{S+1} taps each way, then the even rows and columns), filter the five moments horizontally then
// vertically (N_S taps, valid positions only), and add the per-pixel num and den terms of the tile's valid positions in
// a fixed order into one f64 partial each.
namespace {
template <int S>
constexpr int kVifIn = CCD_SSIM_T + ccd_vif_taps(S) - 1;  // staged rows and columns
template <int S>
constexpr size_t kVifSmem = sizeof(double) * (2 * kVifIn<S> * kVifIn<S> + 5 * kVifIn<S> * CCD_SSIM_T + 2 * kTileWarps);
struct VifArgs {
    double g[17];   // this scale's N_S taps
    double gn[9];   // the next scale's taps
};
}  // namespace

template <int S>
__global__ void __launch_bounds__(32 * kTileWarps, 2) k_frame_vif(const VifJobDev *__restrict__ jobs, const VifArgs a) {
    constexpr int T = CCD_SSIM_T, K = kTileK, N = ccd_vif_taps(S), In = kVifIn<S>;
    extern __shared__ double vif_sm[];
    double *sh = vif_sm;                             // [5][In][T]: the horizontal pass
    double *sx = sh + 5 * In * T, *sy = sx + In * In;  // [In][In]
    double *sred = sy + In * In;                     // [warps][2]
    const VifJobDev &J = jobs[blockIdx.y];
    const int tid = (int)threadIdx.x;
    const auto [c, t, h, w] = locate_tile(J, [](int n) { return ccd_vif_side(n, S); }, ccd_ssim_tiles);
    if (c == 3) return;
    const int tw = (w + T - 1) / T, y0 = t / tw * T, x0 = t % tw * T;

    unsigned long long bad = ~0ull;
    const unsigned n0 = (unsigned)J.h * J.w, n1 = (unsigned)(J.h >> J.cs) * (unsigned)(J.w >> J.cs);
    for (int i = tid; i < In * In; i += 32 * kTileWarps) {
        const int r = i / In, q = i - r * In, y = y0 + r, x = x0 + q;
        double vx = 0.0, vy = 0.0;
        if (y < h && x < w) {
            const unsigned s = (unsigned)y * (unsigned)w + (unsigned)x;
            if constexpr (S == 0) {
                const SamplePair P = read_pair(J, c, s, n0, n1);
                vx = __ddiv_rn(__dmul_rn((double)P.d.kd, 255.0), J.Md);
                vy = __ddiv_rn(__dmul_rn((double)P.ks, 255.0), J.Md);
                if (r < T && q < T && CCD_OFF_GRID(P.d)) bad = min(bad, (unsigned long long)P.pidx);
            } else {
                const double2 v = J.lvl[c][S][s];
                vx = v.x;
                vy = v.y;
            }
        }
        sx[i] = vx;
        sy[i] = vy;
    }
    if constexpr (S == 0) report_bad(bad, J.bad, tid);
    __syncthreads();

    if constexpr (S + 1 < CCD_VIF_SCALES) {  // the next scale: N_{S+1} taps "valid" each way, the even rows and columns
        constexpr int NN = ccd_vif_taps(S + 1);
        const int r = tid / (T / 2), q = tid % (T / 2), Y = (y0 >> 1) + r, X = (x0 >> 1) + q;
        const int hn = (h - NN + 2) >> 1, wn = (w - NN + 2) >> 1;
        if (Y < hn && X < wn) {
            const double *px = sx + 2 * r * In + 2 * q, *py = sy + 2 * r * In + 2 * q;
            double ox = 0.0, oy = 0.0;
#pragma unroll
            for (int u = 0; u < NN; u++) {  // rows first, then the column: the order of the separable restatement
                double hx = 0.0, hy = 0.0;
#pragma unroll
                for (int v = 0; v < NN; v++) {
                    hx = fma(a.gn[v], px[u * In + v], hx);
                    hy = fma(a.gn[v], py[u * In + v], hy);
                }
                ox = fma(a.gn[u], hx, ox);
                oy = fma(a.gn[u], hy, oy);
            }
            J.lvl[c][S + 1][(size_t)Y * wn + X] = make_double2(ox, oy);
        }
    }

    moments_h<N, In>(sx, sy, a.g, sh, tid);
    __syncthreads();

    double s_num = 0.0, s_den = 0.0;
    {
        const int q = tid & 31, r0 = (tid >> 5) * K;
        double m[5][K];
        moments_v<N, In>(sh, a.g, q, r0, m);
        const int x = x0 + q, wo = w - N + 1, ho = h - N + 1;
#pragma unroll
        for (int k = 0; k < K; k++) {
            const int y = y0 + r0 + k;
            if (x >= wo || y >= ho) continue;
            // no contraction: identical images give sigma_ref^2 = sigma_dist^2 = sigma_12 exactly, as in the checker
            const double mu1 = m[1][k], mu2 = m[0][k];  // reference (source), distorted (decoded)
            double s1 = fmax(__dsub_rn(m[3][k], __dmul_rn(mu1, mu1)), 0.0);
            const double s2 = fmax(__dsub_rn(m[2][k], __dmul_rn(mu2, mu2)), 0.0);
            const double s12 = __dsub_rn(m[4][k], __dmul_rn(mu1, mu2));
            double g = __ddiv_rn(s12, __dadd_rn(s1, 1e-10));
            double sv = __dsub_rn(s2, __dmul_rn(g, s12));
            if (s1 < 1e-10) {
                g = 0.0;
                sv = s2;
                s1 = 0.0;
            }
            if (s2 < 1e-10) {
                g = 0.0;
                sv = 0.0;
            }
            if (g < 0.0) {
                sv = s2;
                g = 0.0;
            }
            sv = fmax(sv, 1e-10);
            s_num = __dadd_rn(s_num, log10(__dadd_rn(1.0, __ddiv_rn(__dmul_rn(__dmul_rn(g, g), s1), __dadd_rn(sv, 2.0)))));
            s_den = __dadd_rn(s_den, log10(__dadd_rn(1.0, __ddiv_rn(s1, 2.0))));
        }
    }
    tile_sums(s_num, s_den, sred, tid, [&](double pn, double pd) {
        J.part[S][2 * blockIdx.x] = pn;
        J.part[S][2 * blockIdx.x + 1] = pd;
    });
}

template <int S>
static int vif_launch_scale(const VifJobDev *d_jobs, int n_jobs, int tiles, const double *g, const double *gn,
                            cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_frame_vif<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVifSmem<S>);
    if (e != cudaSuccess) return (int)e;
    VifArgs a;
    memset(&a, 0, sizeof(a));
    memcpy(a.g, g, sizeof(double) * ccd_vif_taps(S));
    if (gn) memcpy(a.gn, gn, sizeof(double) * ccd_vif_taps(S + 1));
    k_frame_vif<S><<<dim3((unsigned)tiles, (unsigned)n_jobs, 1), 32 * kTileWarps, kVifSmem<S>, st>>>(d_jobs, a);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_vif_launch(const VifJobDev *d_jobs, int n_jobs, const int max_tiles[CCD_VIF_SCALES], const double g[CCD_VIF_SCALES][17],
                   cudaStream_t st) {
    // scale s + 1 reads the samples scale s wrote: stream order
    if (int e = vif_launch_scale<0>(d_jobs, n_jobs, max_tiles[0], g[0], g[1], st)) return e;
    if (int e = vif_launch_scale<1>(d_jobs, n_jobs, max_tiles[1], g[1], g[2], st)) return e;
    if (int e = vif_launch_scale<2>(d_jobs, n_jobs, max_tiles[2], g[2], g[3], st)) return e;
    return vif_launch_scale<3>(d_jobs, n_jobs, max_tiles[3], g[3], nullptr, st);
}

// ---- PSNR-HVS-M.  A = the source, B = the decoded image, both in 8-bit units v = k * 255 / M (f64).  Per tile: stage
// the integers of a strip of CCD_HVS_ROWS x CCD_HVS_COLS samples of both images (32 blocks side by side); then one
// thread per (block, row) forms the row's integer sums and its 8-point DCT, and after that one thread per (block,
// column) the column's DCT, masking sum and error sums.  The 8 lanes of a block reduce by a butterfly, which leaves
// the same bits in every lane, and the tile adds its blocks in a fixed order into one f64 partial per sum.
namespace {
constexpr int kHvsLd = CCD_HVS_COLS + 1;  // staged row stride: the 8 rows of a block fall in distinct banks
static_assert(CCD_HVS_ROWS == 8 && CCD_HVS_COLS / 8 * 8 == 32 * kTileWarps, "one thread per (block, row), then per (block, column)");
struct HvsArgs {
    double dct[8][8];  // dct[k][n]: the orthonormal 8-point DCT-II basis, computed on the host
};
// Ponomarenko et al. (2007), rows k = 0..7, columns l = 0..7: CSF = round(25.735088 / Q, 6), Mask = round((10 / Q)^2,
// 6), Q the JPEG luminance quantisation table.  Read through the read-only path: the 8 columns of a warp's lanes share
// one cache line.
__device__ const double kHvsCsf[64] = {
    1.608443, 2.339554, 2.573509, 1.608443, 1.072295, 0.643377, 0.504610, 0.421887,
    2.144591, 2.144591, 1.838221, 1.354478, 0.989811, 0.443708, 0.428918, 0.467911,
    1.838221, 1.979622, 1.608443, 1.072295, 0.643377, 0.451493, 0.372972, 0.459555,
    1.838221, 1.513829, 1.169777, 0.887417, 0.504610, 0.295806, 0.321689, 0.415082,
    1.429727, 1.169777, 0.695543, 0.459555, 0.378457, 0.236102, 0.249855, 0.334222,
    1.072295, 0.735288, 0.467911, 0.402111, 0.317717, 0.247453, 0.227744, 0.279729,
    0.525206, 0.402111, 0.329937, 0.295806, 0.249855, 0.212687, 0.214459, 0.254803,
    0.357432, 0.279729, 0.270896, 0.262603, 0.229778, 0.257351, 0.249855, 0.259950};
__device__ const double kHvsMask[64] = {
    0.390625, 0.826446, 1.000000, 0.390625, 0.173611, 0.062500, 0.038447, 0.026874,
    0.694444, 0.694444, 0.510204, 0.277008, 0.147929, 0.029727, 0.027778, 0.033058,
    0.510204, 0.591716, 0.390625, 0.173611, 0.062500, 0.030779, 0.021004, 0.031888,
    0.510204, 0.346021, 0.206612, 0.118906, 0.038447, 0.013212, 0.015625, 0.026015,
    0.308642, 0.206612, 0.073046, 0.031888, 0.021626, 0.008417, 0.009426, 0.016866,
    0.173611, 0.081633, 0.033058, 0.024414, 0.015242, 0.009246, 0.007831, 0.011815,
    0.041649, 0.024414, 0.016437, 0.013212, 0.009426, 0.006830, 0.006944, 0.009803,
    0.019290, 0.011815, 0.011080, 0.010412, 0.007972, 0.010000, 0.009426, 0.010203};
}  // namespace

// y[k] = sum_n dct[k][n] x[n]: 8 FMAs per output, n in order
static __device__ __forceinline__ void hvs_dct8(const double (&x)[8], const double (&dct)[8][8], double (&y)[8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        double acc = 0.0;
#pragma unroll
        for (int n = 0; n < 8; n++) acc = fma(dct[k][n], x[n], acc);
        y[k] = acc;
    }
}

// vari(Z) = (n sum z^2 - (sum z)^2) / (n - 1) from the exact integer sums s, q of the block's k, in 8-bit units
static __device__ __forceinline__ double hvs_vari(long long s, long long q, int n, double s2) {
    return __dmul_rn(__ddiv_rn((double)(n * q - s * s), (double)(n - 1)), s2);
}

// The masking ratio pop of a block, from row e of its integers k in lane e of the block's 8 lanes: 0 for a flat block,
// else the quadrants' vari (top-left, top-right, bottom-right, bottom-left, added in that order) over the block's.
// Every lane of the 8 gets the same value.
static __device__ __forceinline__ double hvs_pop(const int (&k)[8], int e, double s2) {
    long long v[4] = {0, 0, 0, 0};  // sum k and sum k^2 of the row's left half, then of its right half
#pragma unroll
    for (int n = 0; n < 8; n++) {
        v[(n >> 2) * 2] += k[n];
        v[(n >> 2) * 2 + 1] += (long long)k[n] * k[n];
    }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1)  // rows 0..3, or rows 4..7
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
    long long u[4];  // the other four rows
#pragma unroll
    for (int j = 0; j < 4; j++) u[j] = __shfl_xor_sync(0xffffffffu, v[j], 4);
    const long long s = v[0] + v[2] + u[0] + u[2], q = v[1] + v[3] + u[1] + u[3];
    if (64 * q - s * s == 0) return 0.0;
    const bool top = e < 4;
    const double q00 = hvs_vari(top ? v[0] : u[0], top ? v[1] : u[1], 16, s2);
    const double q01 = hvs_vari(top ? v[2] : u[2], top ? v[3] : u[3], 16, s2);
    const double q10 = hvs_vari(top ? u[0] : v[0], top ? u[1] : v[1], 16, s2);
    const double q11 = hvs_vari(top ? u[2] : v[2], top ? u[3] : v[3], 16, s2);
    return __ddiv_rn(__dadd_rn(__dadd_rn(__dadd_rn(q00, q01), q11), q10), hvs_vari(s, q, 64, s2));
}

static __device__ __forceinline__ double hvs_group_sum(double x) {  // the 8 lanes of a block, xor butterfly
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

__global__ void __launch_bounds__(32 * kTileWarps) k_frame_hvs(const HvsJobDev *__restrict__ jobs, const HvsArgs a) {
    constexpr int R = CCD_HVS_ROWS, W = CCD_HVS_COLS;
    __shared__ double hvs_sm[2 * R * kHvsLd];  // [2][R][kHvsLd]: the staged integers (int), then the row pass (f64)
    __shared__ double sred[2 * kTileWarps];
    int *si = reinterpret_cast<int *>(hvs_sm);
    const HvsJobDev &J = jobs[blockIdx.y];
    const int tid = (int)threadIdx.x;
    const auto [c, t, h, w] = locate_tile(J, [](int n) { return n; }, ccd_hvs_tiles);
    if (c == 3) return;
    const int tw = (w + W - 1) / W, y0 = t / tw * R, x0 = t % tw * W;

    // every sample of the strip, for the off-grid check; rows [0, R) of A (source), then of B (decoded)
    unsigned long long bad = ~0ull;
    const unsigned n0 = (unsigned)J.h * J.w, n1 = (unsigned)(J.h >> J.cs) * (unsigned)(J.w >> J.cs);
    for (int i = tid; i < R * W; i += 32 * kTileWarps) {
        const int r = i / W, q = i % W, y = y0 + r, x = x0 + q;
        int ka = 0, kb = 0;
        if (y < h && x < w) {
            const unsigned s = (unsigned)y * (unsigned)w + (unsigned)x;
            const SamplePair P = read_pair(J, c, s, n0, n1);
            kb = (int)P.d.kd;
            ka = P.ks;
            if (CCD_OFF_GRID(P.d)) bad = min(bad, (unsigned long long)P.pidx);
        }
        si[r * kHvsLd + q] = ka;
        si[(R + r) * kHvsLd + q] = kb;
    }
    report_bad(bad, J.bad, tid);
    __syncthreads();

    const int b = tid >> 3, e = tid & 7;  // this thread's block of the strip, and its row, then its column
    double xa[8], xb[8], ya[8], yb[8];
    double pop_a, pop_b;
    {
        int ka[8], kb[8];
#pragma unroll
        for (int n = 0; n < 8; n++) {
            ka[n] = si[e * kHvsLd + 8 * b + n];
            kb[n] = si[(R + e) * kHvsLd + 8 * b + n];
        }
        __syncthreads();  // the row pass overwrites the staged integers
        pop_a = hvs_pop(ka, e, J.s2);
        pop_b = hvs_pop(kb, e, J.s2);
#pragma unroll
        for (int n = 0; n < 8; n++) {
            xa[n] = __ddiv_rn(__dmul_rn((double)ka[n], 255.0), J.Md);
            xb[n] = __ddiv_rn(__dmul_rn((double)kb[n], 255.0), J.Md);
        }
    }
    hvs_dct8(xa, a.dct, ya);
    hvs_dct8(xb, a.dct, yb);
#pragma unroll
    for (int l = 0; l < 8; l++) {
        hvs_sm[e * kHvsLd + 8 * b + l] = ya[l];
        hvs_sm[(R + e) * kHvsLd + 8 * b + l] = yb[l];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 8; r++) {
        xa[r] = hvs_sm[r * kHvsLd + 8 * b + e];
        xb[r] = hvs_sm[(R + r) * kHvsLd + 8 * b + e];
    }
    hvs_dct8(xa, a.dct, ya);  // ya[k] = A_dct[k][e], yb[k] = B_dct[k][e]
    hvs_dct8(xb, a.dct, yb);

    double m_a = 0.0, m_b = 0.0;  // sum of A_dct^2 Mask over the block but (0, 0)
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const double wm = k == 0 && e == 0 ? 0.0 : __ldg(kHvsMask + 8 * k + e);
        m_a = fma(__dmul_rn(ya[k], ya[k]), wm, m_a);
        m_b = fma(__dmul_rn(yb[k], yb[k]), wm, m_b);
    }
    m_a = hvs_group_sum(m_a);
    m_b = hvs_group_sum(m_b);
    const double T = fmax(__dmul_rn(__dsqrt_rn(__dmul_rn(m_a, pop_a)), 1.0 / 32), __dmul_rn(__dsqrt_rn(__dmul_rn(m_b, pop_b)), 1.0 / 32));
    double s_hvs = 0.0, s_hvs_m = 0.0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const double csf = __ldg(kHvsCsf + 8 * k + e);
        const double u = fabs(__dsub_rn(ya[k], yb[k])), d = __dmul_rn(u, csf);
        s_hvs = fma(d, d, s_hvs);
        const double um = k == 0 && e == 0 ? u : fmax(__dsub_rn(u, __ddiv_rn(T, __ldg(kHvsMask + 8 * k + e))), 0.0);
        const double dm = __dmul_rn(um, csf);
        s_hvs_m = fma(dm, dm, s_hvs_m);
    }
    s_hvs = hvs_group_sum(s_hvs);
    s_hvs_m = hvs_group_sum(s_hvs_m);
    const bool own = e == 0 && y0 + 8 <= h && x0 + 8 * b + 8 <= w;  // lane 0 of a block wholly inside the plane
    if (own && J.map[c]) J.map[c][(size_t)(y0 >> 3) * (w >> 3) + (x0 >> 3) + b] = __double2float_rn(__ddiv_rn(s_hvs_m, 64.0 * 255 * 255));
    s_hvs_m = own ? s_hvs_m : 0.0;
    s_hvs = own ? s_hvs : 0.0;
    tile_sums(s_hvs_m, s_hvs, sred, tid, [&](double pm, double p) {
        J.part[2 * blockIdx.x] = pm;
        J.part[2 * blockIdx.x + 1] = p;
    });
}

int ccd_hvs_launch(const HvsJobDev *d_jobs, int n_jobs, int max_tiles, const double dct[8][8], cudaStream_t st) {
    HvsArgs a;
    memcpy(a.dct, dct, sizeof(a.dct));
    k_frame_hvs<<<dim3((unsigned)max_tiles, (unsigned)n_jobs, 1), 32 * kTileWarps, 0, st>>>(d_jobs, a);
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_finish(const float *d_in, int h, int w, int bitdepth, int data_type, float *a, float *b, float *c,
               cudaStream_t st) {
    const float M = (float)((1 << bitdepth) - 1);
    const size_t n = (size_t)h * w;
    if (data_type != 1) {
        k_finish_444<<<(unsigned)((3 * n + 255) / 256), 256, 0, st>>>(d_in, 3 * n, M, a);
    } else {
        k_finish_444<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_in, n, M, a);
        if (h / 2 > 0 && w / 2 > 0) {
            k_finish_420_uv<<<grid2(w / 2, h / 2, 2), kBlock2, 0, st>>>(d_in, h, w, M, b, c);
            g_ccd_launches++;
        }
    }
    g_ccd_launches++;
    return (int)cudaGetLastError();
}
