// ccd_internal.h -- structures shared between the host API and the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ccdec.h"

// --------------------------------------------------------------------------------------
// Entropy stage (ccd_entropy.cu): one persistent CTA per Cool-chic stream.
// --------------------------------------------------------------------------------------
#define CCD_ENT_THREADS 512          // <= 14 producer warps + helper warp + range-coder warp
#define CCD_ENT_THREADS_NARROW 256   // 5 producer warps + helper + coder: two streams per SM when a call holds more streams than SMs
#define CCD_ENT_WARPS (CCD_ENT_THREADS / 32)
#define CCD_ENT_PRODUCERS (CCD_ENT_WARPS - 2)
#define CCD_WIN 32                   // cumulative-window entries per symbol (31 decodable symbols)
#define CCD_WIN_HALF 14              // window = symbols mu_int-14 .. mu_int+16; the mode sits at the EVEN index 14
                                     // so that (left(mode), left(mode+1)) is one aligned LDS.64
#define CCD_HOT_MIRROR 8            // hot-ring entries duplicated behind the end of the ring
#define CCD_ROW_COLS 64              // row ring: columns kept per row (power of 2)
#define CCD_IFCE_FAST_MAX 12         // IFCE inputs handled by the fast (quad) kernel; more -> generic kernel
#define CCD_MAX_DIM 72               // n_ctx (<=40) + n_ifce_out (<=31)
#define CCD_N_SCALE 2561
#define CCD_MASK_STRIDE 10           // wavefront stride = ARM mask size 9 + 1 (latent.py:63,72)
#define CCD_SMEM_MAX (227 * 1024)    // dynamic shared memory one CTA may use on sm_90

// One latent grid, in DECODE order (index 0 = coarsest = first decoded).
struct EntGrid {
    int32_t h, w;
    int32_t n_diag;        // w + 10*(h-1), or h*w in raster mode
    int32_t raster;        // w <= 9: plain raster scan (latent.py:113-122)
    int64_t lat_off;       // offset of this grid in the latent array (decode order)
    int32_t ifce_in;       // number of IFCE inputs (0: features are zero)
    int32_t ifce_blob_off; // byte offset of this grid's IFCE parameters in the blob
    int32_t ifce_blob_bytes;
    int32_t n_dec;         // grids decoded before this one
    // IFCE input channel c reads grid (this-1-c) at (yy >> sh, xx >> sh); sh < 0: constant 0
    int32_t ch_w[31];
    int32_t ch_sh[31];
    int64_t ch_off[31];
};

// The range decoder between two symbols (DESIGN §4.8): D, R, the next unread word and the first word of the coder's
// register window.  A launch starts from one the host writes (the stream's first two words for a fresh decode, a saved
// one to resume) and stores the one after its last symbol.
struct EntCoderState {
    uint64_t D, R;
    uint32_t wpos, wbase;
    uint32_t slow;         // symbols of the launch decoded with the exact f64 model (stored, not read)
    uint32_t pad;
};

// One launch decodes grid[0 .. n_grids) of a stream: all of its grids, or a range of them in decode order (a stage of
// a progressive decode).  Symbol indices (ord, the control words, the tags) start at 0 in every launch; latents are
// written at each grid's absolute lat_off.
struct EntStream {
    int32_t n_grids;
    int32_t n_ctx, cf, n_hidden, has_ifce;
    int32_t ring;          // window ring entries (power of two)
    int32_t rows;          // row ring rows (power of two)
    int32_t mode;          // 0 decode, 1 encode given latents, 2 sample + encode
    uint32_t prod_mask;    // which of warps 0..13 produce (14 = coder helper, 15 = range coder)
    const uint32_t *words; // compressed words (device)
    int64_t n_words;
    int8_t *latents;       // device, decode order
    int64_t n_symbols;
    const unsigned char *blob; // device: ARM parameters followed by IFCE parameters
    int32_t arm_blob_bytes;
    int32_t ifce_blob_max;     // largest per-grid IFCE blob
    int32_t *status;           // device: [0] error code, [1] words consumed, [2] slow-path count
    uint64_t seed;
    uint32_t *out_words;       // encode modes: output words (device)
    int64_t out_cap;
    EntGrid grid[CCD_MAX_GRIDS];
    // (after the grid table, so that no field before it moves)
    EntCoderState start;       // the decoder's state at the launch's first symbol (decode mode)
    EntCoderState *end;        // device: the state after its last symbol
};

// Blob layouts ---------------------------------------------------------------------------
// FAST (f64 on the DMMA m8n8k4 tensor cores, every value an integer below 2^53: proven by arm_fits_f64); a symbol
// is evaluated by a quad of lanes, member t owning inputs t, t + 4, ...:
//   ks = ceil(dim/4) k-steps, nt = ceil(ks/2) n-tiles; unit(j, c) = 8j + 4(c & 1) + (c >> 1) (column c of tile j)
//   f64 Wh[n_hidden][ks][nt][32]   B fragments: lane L holds W[4s + (L & 3)][unit(j, L >> 2)]
//   f64 Bh[n_hidden][nt][8]        C fragments: column c of tile j holds B[unit(j, c)]
//   f64 Wo[4 ks][4]                last layer (2 outputs), then stabiliser (2 outputs); rows >= dim are zero
//   int64 Bl[2], Bs[2]
// IFCE arm (FAST): int32 W[n_in][cfp] (cfp = cf rounded up to 4), pad8, int64 B[cf]
// GENERIC (all int64): W64h[n_hidden][dim][dim], Wl[dim][2], Ws[dim][2], Bh, Bl, Bs;
//   IFCE: int64 W[n_in][cf], B[cf]

// number of kernels launched by this library since load (bench.py reports it)
extern unsigned long long g_ccd_launches;

struct EntLaunchCfg {
    int n_ctx, cf;   // template selection
    bool fast;
    size_t smem_bytes;
    int threads;     // CCD_ENT_THREADS, or CCD_ENT_THREADS_NARROW for two CTAs per SM
};

int ccd_entropy_launch(const EntStream *d_streams, int n_streams, const EntLaunchCfg &cfg,
                       const uint32_t *d_cdf, const float *d_scale, cudaStream_t st);
size_t ccd_entropy_smem_bytes(int ring, int rows, int arm_blob_bytes, int ifce_blob_max);
bool ccd_entropy_has_fast(int n_ctx, int cf);
int ccd_cdf_table_build(uint32_t *d_cdf, const float *d_scale, cudaStream_t st);
int ccd_laplace_domain(const float *d_scale, int sc_lo, int sc_hi, uint32_t *d_lo, uint32_t *d_hi,
                       cudaStream_t st);

// --------------------------------------------------------------------------------------
// Rate pass (ccd_entropy.cu, after the entropy kernel): the information content of every decoded latent under the
// model the range coder used.  All latents are known, so every symbol's context is known: no wavefront, one CTA
// per tile of CCD_RATE_TH x CCD_RATE_TW symbols of one grid of one job, all jobs in one launch.
// --------------------------------------------------------------------------------------
#define CCD_RATE_THREADS 256
#define CCD_RATE_TH 28               // tile rows; + 4 causal halo rows = the 32-row ring
#define CCD_RATE_TW 56               // tile columns; + 4 halo columns each side = the 64 ring columns
#define CCD_RATE_ROWS 32

struct RateJobDev {
    const EntStream *es;      // device: the job's stream descriptor (grids, ARM blob, latents in decode order)
    float *bits;              // [n_symbols] 24 - log2(freq), decode order
    uint32_t *freq;           // optional
    uint32_t *mu_sc;          // optional: mu_idx | sc_idx << 16
    unsigned long long *bad;  // smallest decode-order index of a latent outside [-64, 63] (~0 if none)
    int32_t kind;             // ARM variant (ccd_rate_kind)
};
struct RateTile {
    int32_t job, grid, y0, x0;  // grid: decode-order index (0 = coarsest)
};
// spatial rate map of one job (finest grid first, canonical fp32 order)
struct RateSpatialDev {
    const float *bits;
    float *out;               // [H][W]
    int32_t H, W, n_grids;
    int32_t h[CCD_MAX_GRIDS], w[CCD_MAX_GRIDS];
    int64_t off[CCD_MAX_GRIDS];   // decode-order offset of the grid in bits
    float ratio[CCD_MAX_GRIDS];   // fp32((H * W) / (h * w))
    float sy[CCD_MAX_GRIDS], sx[CCD_MAX_GRIDS];  // nearest-resize scales h / H, w / W (fp32)
};

// The kind k_entropy and k_latent_rate dispatch on: the shape's index among the fast shapes when fast, else generic
int ccd_rate_kind(int n_ctx, int cf, bool fast);
size_t ccd_rate_smem_bytes(int arm_blob_bytes, int ifce_blob_max);
int ccd_rate_launch(const RateTile *d_tiles, int n_tiles, const RateJobDev *d_jobs, size_t smem, const uint32_t *d_cdf,
                    const float *d_scale, double *d_part, cudaStream_t st);
int ccd_rate_spatial_launch(const RateSpatialDev *d_jobs, int n_jobs, int64_t max_pixels, cudaStream_t st);

// Scale-calibration sweep (k_rate_sweep, DESIGN §4.10): the RateTile list of the rate pass (job = sweep job), one CTA
// per tile.  Each thread holds up to CCD_SWEEP_SPT symbols of its tile; one f64 partial per (tile, offset) in
// part[CCD_SWEEP_MAX_OFFSETS * tile + k]; the grid histograms are integer atomics on counters the host zeroes.
#define CCD_SWEEP_SPT ((CCD_RATE_TH * CCD_RATE_TW + CCD_RATE_THREADS - 1) / CCD_RATE_THREADS)
struct SweepJobDev {
    const int8_t *lat;            // decoded latents, decode order
    const uint32_t *mu_sc;        // mu_idx | sc_idx << 16, same layout
    unsigned long long *hist;     // [n_grids][128], decode-order grids
    unsigned long long *bad;      // smallest decode-order index of a bad symbol (~0 if none)
    int32_t n_off;
    int32_t off[CCD_SWEEP_MAX_OFFSETS];
    int32_t h[CCD_MAX_GRIDS], w[CCD_MAX_GRIDS];  // decode order
    int64_t lat_off[CCD_MAX_GRIDS];
};
int ccd_rate_sweep_launch(const RateTile *d_tiles, int n_tiles, const SweepJobDev *d_jobs, const uint32_t *d_cdf,
                          const float *d_scale, double *d_part, cudaStream_t st);

// Candidate pricing (k_rate_candidates, DESIGN §4.11): the RateTile list of the rate pass for one job, one CTA per
// tile.  Candidate 0 is the model itself; candidate k > 0 changes ONE fixed-point weight or bias of the ARM or of one
// grid's IFCE by dv (the change build_arm makes of a change of one transmitted integer).  One f64 partial per
// (tile, candidate) in part[n_cand * tile + k], summed in the order of the rate kernel the edited model takes.
enum { CCD_CAND_BASE = 0, CCD_CAND_ARM = 1, CCD_CAND_STAB = 2, CCD_CAND_IFCE = 3 };
struct CandDev {
    int32_t type;        // CCD_CAND_*
    int32_t l;           // ARM: layer (n_hidden = the output layer); IFCE: the decode-order grid
    int32_t i;           // ARM: input, IFCE: channel of a weight; -1: a bias
    int32_t o;           // ARM: unit, IFCE: feature
    int64_t dv;          // change of the fixed-point weight / bias
    int32_t quad_order;  // 1: the fast rate kernel's summation order (a quad of lanes per symbol), 0: the generic's
    int32_t pad;
};
struct CandJobDev {
    const EntStream *es;      // GENERIC (int64) ARM and IFCE blobs whatever the decoder's kernel
    unsigned long long *bad;  // smallest decode-order index of a latent outside [-64, 63] (~0 if none)
    int32_t n_cand;           // candidates + 1
};
// bytes of dynamic shared memory of k_rate_candidates for a job
size_t ccd_rate_candidates_smem_bytes(int arm_blob_bytes, int ifce_blob_max, int n_cand);
// wide: an ARM wider than 32 or deeper than 3 hidden layers (the kernel's per-thread arrays are sized for it)
int ccd_rate_candidates_launch(const RateTile *d_tiles, int n_tiles, const CandJobDev *d_job, const CandDev *d_cand,
                               bool wide, size_t smem, const uint32_t *d_cdf, const float *d_scale, double *d_part,
                               cudaStream_t st);

// --------------------------------------------------------------------------------------
// Synthesis stage (ccd_synth.cu)
// --------------------------------------------------------------------------------------
struct SynLayerDev {
    int cin, cout, k, residual, relu;
    const float *w; // [cout][cin][k][k]
    const float *b; // [cout]
};

int ccd_ups_pre(const int8_t *d_lat, int h, int w, const float *w1d, int k, float *d_out, cudaStream_t st);
int ccd_ups_first(const int8_t *d_lat, int h, int w, float *d_out, cudaStream_t st);
int ccd_ups_convt(const float *d_in, int c, int h, int w, const float *w1d, int k, float *d_out, int ht,
                  int wt, cudaStream_t st);
// one cascade level in one launch (ups_k == 8, ups_pre_k == 7 only): out[0] = pre-concat conv of the target latent,
// out[1 + c] = transposed conv of in[c]
int ccd_ups_level(const int8_t *d_lat, int th, int tw, const float *d_in, int cc, int ch, int cw, const float *wt1d,
                  const float *wc1d, float *d_out, cudaStream_t st);
int ccd_syn_layer(const float *d_in, int h, int w, const SynLayerDev &L, float *d_out, cudaStream_t st);
int ccd_syn_pointwise2(const float *d_in, int h, int w, const SynLayerDev &L0, const SynLayerDev &L1,
                       float *d_out, cudaStream_t st);
// The synthesis architectures that k_syn_fused and k_tail_syn evaluate in one kernel: 1x1 cin -> hid (cin <= 16,
// hid <= 256), 1x1 hid -> C (C in 2..5), 0-2 3x3 layers C -> C, the stabiliser (if any) 1x1 <= cin -> C, the output
// transform 1x1 C -> C.
bool ccd_syn_fused_family(int cin, const SynLayerDev *layers, int n_layers, const SynLayerDev *stab,
                          const SynLayerDev &ot);
// whole synthesis in one kernel when the architecture is in the fused family (returns -1 otherwise: use the layer
// kernels)
int ccd_syn_fused(const float *d_in, int h, int w, int cin, const SynLayerDev *layers, int n_layers,
                  const SynLayerDev *stab, const SynLayerDev &ot, float *d_out, cudaStream_t st);
int ccd_syn_add(float *d_a, const float *d_b, size_t n, cudaStream_t st);

// ---- batched float tail (ccd_synth.cu): device-resident job arrays, one launch per cascade level and one for
// the last level + synthesis + frame tail of ALL streams of a group (a synthesis in the fused family)
struct CcdTailSynDesc {
    const int8_t *lat;        // finest latent grid [h][w]
    const float *stk;         // coarser stack [cin - 1][ch][cw] (fp32), or ...
    const int8_t *stk8;       // ... the coarsest latent itself when the stream has two grids
    float *out[5];            // output planes
    int h, w, ch, cw, cin;
    const SynLayerDev *layers;
    int n_layers;
    const SynLayerDev *stab;  // may be null
    SynLayerDev ot;
    int finish;               // 0 raw, 1 frame tail (full planes), 2 frame tail 4:2:0
    float M;
    const float *wt1d, *wc1d; // 8 / 7 taps of the last cascade level
    int allow_tma;
};
size_t ccd_tail_job_bytes(void);
size_t ccd_tail_level_job_bytes(void);
void ccd_tail_fill_level(void *dst, const int8_t *lat, const float *in, const int8_t *in8, float *out, int cc, int ch,
                         int cw, int th, int tw, const float *wt1d, const float *wc1d);
int ccd_tail_launch_level(const void *d_jobs, int n_jobs, int planes, int max_tw, int max_th, cudaStream_t st);
void ccd_tail_fill_syn(void *dst, const CcdTailSynDesc &T);
int ccd_tail_launch_syn(const void *d_jobs, int n_jobs, int cinp, int C, int n3_max, int hid_max, int max_w, int max_h,
                        cudaStream_t st);
int ccd_resize_nearest(const float *d_in, int c, int h, int w, float *d_out, int H, int W, cudaStream_t st);
// F.interpolate bilinear (mode 1) / bicubic (mode 2), align_corners=False; sy/sx = 0.5 (scale_factor 2) or in/out
int ccd_resize_torch(const float *d_in, int c, int h, int w, float *d_out, int H, int W, int mode, float sy, float sx,
                     cudaStream_t st);
// samples [first, first+n) of the common-randomness generator (noise.py)
int ccd_cr_noise(float *d_out, size_t first, size_t n, cudaStream_t st);
// canonical sin / cos / log (fn 0 / 1 / 2, ccd_detmath.h) of n doubles
int ccd_detmath(int fn, const double *d_x, double *d_y, size_t n, cudaStream_t st);
// the taps of the windowed-sinc warp (N = taps in {6, 8, ..., 14}) at n offsets: d_c[N i + k]; -1 for another N
int ccd_sinc_coeffs(int taps, const float *d_s, float *d_c, size_t n, cudaStream_t st);
int ccd_finish(const float *d_in, int h, int w, int bitdepth, int data_type, float *a, float *b, float *c,
               cudaStream_t st);
// The sample operations of decode_frame's frame tail (bitstream/decode.py:191-206), for k_finish_*, the epilogue of
// k_tail_syn and that of k_inter_predict: round to the k / M grid (M = 2^bitdepth - 1), clamp to [0, 1].
static __device__ __forceinline__ float quant(float v, float M) { return __fdiv_rn(rintf(__fmul_rn(M, v)), M); }
static __device__ __forceinline__ float clamp01(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }

int ccd_pack(const float *const planes[3], int h, int w, int cs, int bitdepth, int sample_bytes, int interleaved,
             void *d_out, cudaStream_t st);
int ccd_pack_flat(const float *d_in, size_t n, int bitdepth, int sample_bytes, void *d_out, cudaStream_t st);

// A finished frame and its source samples, as every metric against the source reads them (ccd_synth.cu, next to the
// packing kernels): the first part of DistJobDev, SsimJobDev, VifJobDev and HvsJobDev.
struct FramePairDev {
    const float *p[3];          // finished planes (FrameData layout); planes 1, 2 are [h >> cs][w >> cs]
    const void *src;            // source samples, uint8 (bitdepth <= 8) or uint16: planar, or [h][w][3] when hwc
    int32_t h, w, cs, hwc;
    int32_t wide;               // 2-byte source samples
    float M;                    // 2^b - 1
    unsigned long long *bad;    // smallest planar index of an off-grid decoded sample (~0 if none)
};

// Distortion: one launch for every job of a call, blockIdx.y = job.
struct DistJobDev : FramePairDev {
    float *map;                 // optional [h][w] error map
    float M2;                   // fp32(M^2)
    unsigned long long *sse;    // [3], zeroed by the host
    unsigned int *max_abs;      // [3], zeroed by the host
};
int ccd_dist_launch(const DistJobDev *d_jobs, int n_jobs, int64_t max_pixels, int n_sm, cudaStream_t st);

// A decoded sample read back to its integer kd = rint(v * M) (read_pair in ccd_synth.cu)
struct DecodedSample {
    float v, vm, kd;  // the decoded value, fp32(v * M), rint(v * M)
};
static __device__ __forceinline__ DecodedSample read_decoded(const float *p, unsigned j, float M) {
    const float v = __ldg(p + j), vm = __fmul_rn(v, M);
    return DecodedSample{v, vm, rintf(vm)};
}
// A decoded sample off the k / M grid: outside [0, 1] or more than 1/16 away.  A macro, not a function: written into
// the condition of its if, it compiles to the same branches as k_frame_dist had before it was shared.
#define CCD_OFF_GRID(D) (!((D).v >= 0.0f && (D).v <= 1.0f) || fabsf(__fsub_rn((D).vm, (D).kd)) > 0.0625f)

// Source sample k as uploaded (uint8, or uint16 when wide), never widened on the host
static __device__ __forceinline__ int source_sample(const void *src, bool wide, size_t k) {
    return wide ? (int)__ldg(static_cast<const uint16_t *>(src) + k) : (int)__ldg(static_cast<const uint8_t *>(src) + k);
}

// MS-SSIM (DESIGN §4.6): one k_frame_ssim launch per scale for every plane of every job of a call, blockIdx.y = job,
// blockIdx.x = tile over the job's planes (plane 0's tiles, then plane 1's, then plane 2's, each row-major).  A tile owns
// CCD_SSIM_T x CCD_SSIM_T samples of its plane's level (even origin) and reads a CCD_SSIM_HALO halo below and right.
#define CCD_SSIM_T 32
#define CCD_SSIM_HALO 10
#define CCD_SSIM_SCALES 5
struct SsimJobDev : FramePairDev {
    float *map[3];              // optional scale-0 SSIM maps, [h_c - 10][w_c - 10]
    uint2 *lvl[3][CCD_SSIM_SCALES];  // pyramid levels 1..4 per plane: (decoded, source) 2 x 2 sums of the level above
    double *part[CCD_SSIM_SCALES];   // per scale: (sum cs, sum l cs) of each of the job's tiles, in tile order
    double C1, C2;              // (0.01 M)^2, (0.03 M)^2
};
// tiles of one plane of h x w samples at some level
static __host__ __device__ __forceinline__ int ccd_ssim_tiles(int h, int w) {
    return ((h + CCD_SSIM_T - 1) / CCD_SSIM_T) * ((w + CCD_SSIM_T - 1) / CCD_SSIM_T);
}
// five launches; max_tiles[j]: the most tiles of one job at scale j; g: the 11 Gaussian taps
int ccd_ssim_launch(const SsimJobDev *d_jobs, int n_jobs, const int max_tiles[CCD_SSIM_SCALES], const double g[11],
                    cudaStream_t st);

// VIF (DESIGN §4.12): one k_frame_vif<s> launch per scale, tiles as for MS-SSIM (ccd_ssim_tiles over the plane at scale
// s); a tile stages CCD_SSIM_T + N_s - 1 rows and columns of both images and writes its share of scale s + 1.
#define CCD_VIF_SCALES 4
struct VifJobDev : FramePairDev {
    double2 *lvl[3][CCD_VIF_SCALES];  // scales 1..3 per plane: (decoded, source) in 8-bit units
    double *part[CCD_VIF_SCALES];     // per scale: (sum num, sum den) of each of the job's tiles, in tile order
    double Md;                  // M in f64: a sample k is v = k * 255 / M
};
// the window of scale s: N_s = 2^(4 - s) + 1 taps
static __host__ __device__ __forceinline__ constexpr int ccd_vif_taps(int s) { return (1 << (4 - s)) + 1; }
// a side of n samples at scale 0 is this many at scale s: filtered "valid" with N_s taps, then every other sample
static __host__ __device__ __forceinline__ int ccd_vif_side(int n, int s) {
    for (int t = 1; t <= s; t++) n = (n - ccd_vif_taps(t) + 2) >> 1;
    return n;
}
// four launches; max_tiles[s]: the most tiles of one job at scale s; g[s]: the N_s taps of scale s
int ccd_vif_launch(const VifJobDev *d_jobs, int n_jobs, const int max_tiles[CCD_VIF_SCALES], const double g[CCD_VIF_SCALES][17],
                   cudaStream_t st);

// PSNR-HVS-M (DESIGN §4.13): one k_frame_hvs launch for every plane of every job of a call, tiles laid out as for
// MS-SSIM.  A tile is a strip of CCD_HVS_ROWS rows and CCD_HVS_COLS columns of its plane; the tiles cover every sample
// (each is read once, for the off-grid check), and only the 8 x 8 blocks that lie wholly inside the plane are measured.
#define CCD_HVS_ROWS 8
#define CCD_HVS_COLS 256
struct HvsJobDev : FramePairDev {
    float *map[3];              // optional [h_c >> 3][w_c >> 3]: each block's S_hvs_m / 64 / 255^2
    double *part;               // (sum S_hvs_m, sum S_hvs) of each of the job's tiles, in tile order
    double Md;                  // M in f64: a sample k is v = k * 255 / M
    double s2;                  // (255 / M)^2: integer variances to 8-bit units
};
// tiles of one plane of h x w samples
static __host__ __device__ __forceinline__ int ccd_hvs_tiles(int h, int w) {
    return ((h + CCD_HVS_ROWS - 1) / CCD_HVS_ROWS) * ((w + CCD_HVS_COLS - 1) / CCD_HVS_COLS);
}
// one launch; max_tiles: the most tiles of one job; dct[k][n]: the orthonormal 8-point DCT-II basis
int ccd_hvs_launch(const HvsJobDev *d_jobs, int n_jobs, int max_tiles, const double dct[8][8], cudaStream_t st);

// P/B reconstruction (ccd_inter.cu); returns -1 for an unsupported filter size
struct InterLaunch {
    const float *residue, *motion;  // [4|5][h][w], [2|4][h][w]
    const float *ref0[3], *ref1[3]; // planes of the references; ref1 all null for a P frame
    int ref_cs;                     // 1: reference chroma planes are [h/2][w/2] (4:2:0), 0: full size
    int h, w, is_b;
    int32_t gf[4];                  // global flow (x, y) per reference
    int filter_size;
    float M;                        // 0: pre-rounding output; 2^bitdepth - 1: finished frame (decode.py:191-206)
    int out_420;                    // finished output with [h/2][w/2] chroma planes
    float *out[3];
};
int ccd_inter_launch(const InterLaunch &a, cudaStream_t st);
// P/B prediction statistics (k_inter_stats): the prediction of k_inter_predict, its blending weights and, with a
// source, the squared errors of the prediction and of the reference average.  One f64 partial per CTA and per sum
// (alpha, beta, pred SSE, dummy SSE) in d_part[4 * n_ctas]; ccd_inter_stats_ctas gives n_ctas.
struct InterStatsOut {
    const void *src;                // optional source samples (planar or [h][w][3]), layout of the frame
    int src_hwc, src_wide;
    float src_M;
    float *alpha, *beta, *pred;     // optional maps: [h][w], [h][w], [3][h][w]
    double *part;
};
int64_t ccd_inter_stats_ctas(int h, int w);
int ccd_inter_stats_launch(const InterLaunch &a, const InterStatsOut &o, cudaStream_t st);
// Motion analysis (k_inter_analysis, DESIGN §4.9): the finished frame of every variant (CCD_INTER_VARIANTS, in the
// order of ccdec.h) against the source as k_frame_dist compares it, and the flow statistics of each reference.
// Integer results (sse, max bits, outside, bad) are atomics on counters the host sets; the f64 flow sums are one
// partial per CTA (ccd_inter_stats_ctas of them), d_part[6 * cta + 3 * r + k] for reference r and sum k.
struct InterAnalysisOut {
    const void *src;                // source samples (planar, or [h][w][3] for 4:4:4), layout of the frame
    int src_hwc, src_wide;
    float *flow[2];                 // optional [2][h][w] total displacement per reference
    unsigned long long *sse;        // [CCD_INTER_VARIANTS][3], zeroed
    unsigned long long *max_bits;   // [2] bits of the f64 max |local flow|, zeroed
    unsigned long long *outside;    // [2], zeroed
    unsigned long long *bad;        // smallest pixel index with a non-finite flow (~0 if none)
    double *part;
};
int ccd_inter_analysis_launch(const InterLaunch &a, const InterAnalysisOut &o, cudaStream_t st);
