/* ccoracle.h -- CPU restatement ("oracle") of the Cool-chic 5.0.1 decode path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  Every function cites the reference file:line it restates (paths are
 * relative to the reference checkout).
 *
 * Parity status: PINNED.  The restatement reproduces, for samples/bitstreams/kodim14.cool,
 * the latents (sha256 edade69c...) and the uint8 image produced by the reference's own code
 * run through oracle/refshim (see oracle/gen_golden_kodim14.py, tests/golden/).
 * The range coder arithmetic is third-party (constriction==0.4.2, requirements.txt:10,
 * source not in the reference tree): restated from its published algorithm, pinned by the
 * real-constriction stream kodim14.cool (self-synchronising: 7738 words, no desync) and by
 * byte-exact re-encoding of that stream (tests/test_oracle.py).
 */
#ifndef CCORACLE_H
#define CCORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCO_MAX_GRIDS 32 /* n_latent_grids is a 5-bit field (header.py:268) */
#define CCO_MAX_SYN 8    /* n_layer_synthesis is a 3-bit field (header.py:249) */

/* Layout-identical to CcdCoolChicDesc of include/ccdec.h (checked by tests through
 * cco_sizeof_desc()).  Filled by the host-side header parser from a CoolChicHeader
 * (header.py:243-377) + CoolChicEncoderParameter.__post_init__ (core/coolchic.py:149-225). */
typedef struct CcoDesc {
    int32_t img_h, img_w;
    int32_t n_grids;                    /* incl. hyperlatents; index 0 = finest */
    int32_t grid_h[CCO_MAX_GRIDS];
    int32_t grid_w[CCO_MAX_GRIDS];
    int32_t grid_is_hyper[CCO_MAX_GRIDS];
    int32_t grid_ifce_in[CCO_MAX_GRIDS]; /* input_features_ifce, 0 = no IFCE for this grid */
    int32_t latent_res_lo, latent_res_hi;
    int32_t n_ctx;                      /* spatial_context_arm */
    int32_t n_ifce_out;                 /* output_feature_ifce if flag_ifce else 0 */
    int32_t arm_hidden;                 /* n_hidden_layers_arm */
    int32_t arm_stab;                   /* linear_stabiliser_arm */
    int32_t ups_k, ups_pre_k;
    int32_t n_ups;                      /* = latent_resolution[1] kernels of each kind */
    int32_t n_syn_layers;
    int32_t syn_out[CCO_MAX_SYN];
    int32_t syn_k[CCO_MAX_SYN];
    int32_t syn_res[CCO_MAX_SYN];       /* 1 = residual */
    int32_t syn_relu[CCO_MAX_SYN];      /* 1 = relu */
    int32_t syn_stab;                   /* linear_stabiliser_synth */
    int32_t syn_in;                     /* input_feature_synthesis */
    int32_t common_randomness;
    int32_t final_ups;                  /* 0 nearest, 1 bilinear, 2 bicubic */
    int32_t qshift[8];  /* log2(q_step): arm.w arm.b ifce.w ifce.b ups.w ups.b syn.w syn.b */
    int32_t expgol[8];  /* exp-Golomb order, same indexing */
    int32_t nn_n_bit_pad;
    int32_t flag_ifce;  /* ifce_resolution is not None */
} CcoDesc;

enum {
    CCO_OK = 0,
    CCO_ERR_ARG = -1,
    CCO_ERR_NN_TRUNCATED = -2,
    CCO_ERR_DESYNC = -3, /* range decoder quantile >= 2^24: invalid compressed data */
    CCO_ERR_UNSUPPORTED = -4,
    CCO_ERR_NOMEM = -5
};

int cco_sizeof_desc(void);
int cco_set_threads(int n); /* returns the number of threads the float tail will use */

/* number of NN integers transmitted: counts[m*2+wb] with m in arm,ifce,ups,syn. */
int64_t cco_nn_counts(const CcoDesc *d, int64_t counts[8]);

/* exp-Golomb decode of the NN payload (neuralnet/expgolomb.py:74-130). Returns count or <0. */
int64_t cco_decode_nn(const CcoDesc *d, const uint8_t *bytes, size_t nbytes, int64_t *out,
                      size_t cap);
/* exp-Golomb encode (expgolomb.py:15-71). Returns nbytes (or <0); *n_pad = front padding bits. */
int64_t cco_encode_nn(const CcoDesc *d, const int64_t *ints, size_t n, uint8_t *out, size_t cap,
                      int32_t *n_pad);

/* total number of latent symbols and per-grid offsets in DECODE order (coarsest first). */
int64_t cco_latent_layout(const CcoDesc *d, int64_t offsets[CCO_MAX_GRIDS]);

/* Entropy decode all grids (component/coolchic.py:72-166, latent.py:18-187, armint.py).
 * latents_out: int8, decode order (grid n-1 first), each grid row-major.
 * stats (optional, 8 x int64): [0] words consumed, [1] max|acc|, [2] max|hidden|, [3] n diagonals */
int cco_decode_latents(const CcoDesc *d, const int64_t *nn, const uint8_t *latent_bytes,
                       size_t nbytes, int8_t *latents_out, int64_t *stats);

/* Range ENcode given latents (the mode=="encode" branch of the same functions,
 * rangecoder.py:46-78).  Returns nbytes written or <0; CCO_ERR_ARG for a latent outside
 * [-64, 63].  A symbol costs at most 24.0057 bits: cap >= 4 * (ceil(n * 24.0057 / 32) + 3). */
int64_t cco_encode_latents(const CcoDesc *d, const int64_t *nn, const int8_t *latents,
                           uint8_t *out, size_t cap);

/* Draw latents from the stream's own ARM (quantised Laplace, seeded splitmix64) and
 * encode them -> self-consistent synthetic stream (SURVEY 8d).  Returns nbytes or <0. */
int64_t cco_sample_latents(const CcoDesc *d, const int64_t *nn, uint64_t seed, int8_t *latents_out,
                           uint8_t *out, size_t cap);

/* Upsampling (train-mode kron form, upsampling.py:189-196,312-325,463-500) + Synthesis
 * (synthesis.py:61-76,272-294) + final interpolate/crop (component/coolchic.py:187-192).
 * out: float32 [C_out][img_h][img_w] raw synthesis output.  dense_opt: optional
 * [syn_in][h0][w0] dense latent (synthesis input). */
int cco_synthesize(const CcoDesc *d, const int64_t *nn, const int8_t *latents, float *out,
                   float *dense_opt);

/* F.interpolate(align_corners=False) of [c][h][w] to [c][H][W]; mode 1 bilinear, 2 bicubic;
 * scale_factor_2: the call gave scale_factor=2.0 (scale 0.5) instead of a size. */
int cco_resize(const float *in, int c, int h, int w, float *out, int H, int W, int mode,
               int scale_factor_2);
/* common-randomness synthesis input (noise.py + fixed_upsampling bicubic): out [n][img_h][img_w] */
int cco_cr_noise(const CcoDesc *d, float *out);
/* samples [first, first + n) of the common-randomness generator (noise.py:18-34), before any resize */
int cco_noise_samples(uint64_t first, size_t n, float *out);
/* the canonical functions of detmath.h: y[i] = sin / cos / log (fn 0 / 1 / 2) of x[i] */
int cco_detmath(int fn, const double *x, double *y, size_t n);
/* taps of the windowed sinc warp (warp.py:226-268), N = taps in {6, 8, ..., 14}: c[N i + k] for offset s[i] */
int cco_sinc_coeffs(int taps, const float *s, float *c, size_t n);

/* decode_frame tail for I frames (bitstream/decode.py:191-206): round -> (444->420 avg pool)
 * -> clamp -> round.  data_type 0 rgb, 1 yuv420, 2 yuv444.  in: [3][H][W]; out planes:
 * rgb/444: out_a [3][H][W];  420: out_a = y [H][W], out_b = u, out_c = v [H/2][W/2]. */
int cco_finish_frame(const float *in, int h, int w, int bitdepth, int data_type, float *out_a,
                     float *out_b, float *out_c);

/* P/B prediction (bitstream/decode.py:156-189, intercoding/warp.py:294-397,
 * globalmotion.py:151-160).  residue [4 or 5][H][W], motion [2 or 4][H][W] raw synthesis
 * outputs; ref0/ref1 [3][H][W] (444, already converted); out [3][H][W] pre-rounding. */
int cco_inter_predict(const float *residue, const float *motion, const float *ref0,
                      const float *ref1, int h, int w, int is_b, const int32_t *global_flow,
                      int warp_filter_size, float *out);

/* --- constriction stand-in primitives (for oracle/refshim) ------------------------------ */
void *cco_rc_dec_new(const uint32_t *words, size_t n);
void cco_rc_dec_free(void *h);
int cco_rc_decode_block(void *h, const float *mu, const float *scale, int n, int32_t *out);
uint32_t cco_laplace_left(int s, float mu, float scale);
void cco_laplace_domain(int sc_lo, int sc_hi, uint32_t *lo, uint32_t *hi);

#ifdef __cplusplus
}
#endif
#endif
