/* ccdec.h -- C-ABI of libccdec.so, the H100-native (sm_90a) Cool-chic 5.0 decoder.
 *
 * Drop-in boundary for the DECODE path of Orange-OpenSource/Cool-Chic.  The reference is
 * pure Python and has no FFI of its own; each entry point below names the reference
 * function it replaces (paths relative to the reference checkout).  Host language above
 * this ABI is Python (ctypes, cool-chic_b200/_native.py), mirroring the reference's
 * decode_video / decode_frame / encode_decode_coolchic operator interface; see
 * INTEGRATION.md for the stub a reference maintainer would add.
 *
 * Conventions: plain pointers and sizes, no torch types.  Every function returns an int
 * status (0 = CCD_OK, negative = error, never throws); ccd_last_error() gives the message.
 * "d_" pointers are DEVICE pointers owned by the caller (e.g. torch.empty(..., device="cuda")
 * .data_ptr()); other pointers are HOST memory borrowed for the duration of the call.
 * One CcdContext per device; calls on one context must be serialised by the caller.
 * There is NO CPU fallback: without a CUDA device ccd_create() fails.
 */
#ifndef CCDEC_H
#define CCDEC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCD_VERSION 100 /* 0.1.0 */
#define CCD_MAX_GRIDS 32 /* n_latent_grids: 5-bit header field (bitstream/header/header.py:268) */
#define CCD_MAX_SYN 8    /* n_layer_synthesis: 3-bit header field (header.py:249) */

/* Architecture of one Cool-chic, as parsed from CoolChicHeader (header.py:243-377) and
 * derived like CoolChicEncoderParameter.__post_init__ (component/core/coolchic.py:149-225).
 * Grid index 0 is the finest grid (size_per_latent order). */
typedef struct CcdCoolChicDesc {
    int32_t img_h, img_w;
    int32_t n_grids;
    int32_t grid_h[CCD_MAX_GRIDS];
    int32_t grid_w[CCD_MAX_GRIDS];
    int32_t grid_is_hyper[CCD_MAX_GRIDS];
    int32_t grid_ifce_in[CCD_MAX_GRIDS];
    int32_t latent_res_lo, latent_res_hi;
    int32_t n_ctx;
    int32_t n_ifce_out;
    int32_t arm_hidden;
    int32_t arm_stab;
    int32_t ups_k, ups_pre_k;
    int32_t n_ups;
    int32_t n_syn_layers;
    int32_t syn_out[CCD_MAX_SYN];
    int32_t syn_k[CCD_MAX_SYN];
    int32_t syn_res[CCD_MAX_SYN];
    int32_t syn_relu[CCD_MAX_SYN];
    int32_t syn_stab;
    int32_t syn_in;
    int32_t common_randomness;
    int32_t final_ups; /* 0 nearest, 1 bilinear, 2 bicubic */
    int32_t qshift[8]; /* log2(q_step): arm.w arm.b ifce.w ifce.b ups.w ups.b syn.w syn.b */
    int32_t expgol[8];
    int32_t nn_n_bit_pad;
    int32_t flag_ifce;
} CcdCoolChicDesc;

enum {
    CCD_OK = 0,
    CCD_ERR_ARG = -1,          /* bad argument / inconsistent descriptor */
    CCD_ERR_NN_TRUNCATED = -2, /* NN payload shorter than announced */
    CCD_ERR_DESYNC = -3,       /* range decoder quantile >= 2^24: corrupt latent payload */
    CCD_ERR_UNSUPPORTED = -4,  /* valid syntax the device path does not implement yet */
    CCD_ERR_NOMEM = -5,
    CCD_ERR_CUDA = -6,         /* CUDA runtime error (message in ccd_last_error) */
    CCD_ERR_NO_DEVICE = -7
};

typedef struct CcdContext CcdContext;

int ccd_version(void);
int ccd_sizeof_desc(void);
/* message of the last failing call on this thread (ctx may be NULL) */
const char *ccd_last_error(const CcdContext *ctx);

/* Creates the per-device context: allocates scratch, uploads the normative scale table
 * (bitstream/component/mu_scale.npy, constants.py:24-37) and builds the device-resident
 * quantised-Laplace cumulative table (replaces constriction's per-symbol f64 CDF
 * evaluation, call site rangecoder.py:93). */
int ccd_create(int device_ordinal, CcdContext **out);
void ccd_destroy(CcdContext *ctx);

/* number of transmitted NN integers / latent symbols for a descriptor */
int64_t ccd_nn_count(const CcdCoolChicDesc *desc);
int64_t ccd_latent_count(const CcdCoolChicDesc *desc, int64_t offsets_by_grid[CCD_MAX_GRIDS]);

/* Host-side exp-Golomb decode of the NN payload.
 * Replaces decode_network + decode_exp_golomb (bitstream/neuralnet/neuralnet.py:92-204,
 * bitstream/neuralnet/expgolomb.py:74-130).  Returns the count or a negative status. */
int64_t ccd_decode_nn(const CcdCoolChicDesc *desc, const uint8_t *nn_bytes, size_t nn_nbytes,
                      int64_t *out_ints, size_t cap);

/* One independent Cool-chic to decode.  d_out: float32 [C_out][img_h][img_w] raw synthesis
 * output (un-clamped, un-rounded -- what encode_decode_coolchic returns).  d_latents
 * (optional, may be NULL): int8 decoded latents in decode order (coarsest grid first, each
 * grid row-major).  status (out): per-job status written on completion.
 * Frame tail (optional, the Cool-chic of an I frame, 3 output channels): finish_bitdepth != 0 asks
 * for decode_frame's round / (4:2:0 average) / clamp / round (bitstream/decode.py:191-206), applied
 * by the library -- fused into the synthesis kernel's epilogue where the batched path takes the job:
 * d_out then receives the FINISHED frame -- [3][H][W] for finish_type 0 (rgb), 2 (yuv444),
 * 3 (flow); for finish_type 1 (yuv420) d_out = y [H][W], d_out_u, d_out_v [H/2][W/2].
 *
 * Progressive decoding (DESIGN §4.8): grid_end (0: all grids) stops the entropy stage after the first grid_end grids in
 * decode order (coarsest first).  The output is then the PREVIEW: every grid not yet decoded is read as zeros, exactly
 * what ccd_synthesize_many writes with those grids in zero_grids (frame tail included).  state (NULL: start from the
 * first grid) lets a later call carry on: read on entry, it says where to start (grids_done); on success it is updated
 * to grid_end.  The decoded grids then stay in d_latents, which must be the caller's and is passed again unchanged:
 * the next call reads the coarser grids from it and writes only the grids it decodes.  Decoding the stages one after
 * the other gives latents and an output identical to one call, whatever the split points.  CCD_ERR_ARG, before any
 * launch: grid_end outside (grids_done, n_grids], a state without d_latents, a state of another stream. */
typedef struct CcdEntropyState {
    int32_t grids_done;      /* decode-order grids already in d_latents; 0 for a fresh decode */
    int32_t reserved;
    int64_t words_consumed;  /* payload words the decoded grids needed (a payload cut there decodes them alike) */
    uint64_t opaque[6];      /* the range decoder's state at that boundary and the stream it belongs to */
} CcdEntropyState;

typedef struct CcdJob {
    const CcdCoolChicDesc *desc;
    const uint8_t *nn_bytes;
    size_t nn_nbytes;
    const uint8_t *latent_bytes;
    size_t latent_nbytes;
    float *d_out;
    int8_t *d_latents;
    int32_t status;
    int32_t finish_bitdepth;
    int32_t finish_type;
    float *d_out_u;
    float *d_out_v;
    int32_t grid_end;
    CcdEntropyState *state;
} CcdJob;

/* Decode n independent Cool-chics concurrently (one persistent CTA per stream for the
 * entropy stage, whole-GPU kernels for upsampling + synthesis).  Synchronous w.r.t. the
 * host: returns once results are in device memory.  Replaces, per job,
 * encode_decode_coolchic(mode="decode") (bitstream/component/coolchic.py:29-207), i.e.
 * arm_to_fixed_point_param (armint.py:30-170), the IFCE + wavefront ARM + range-decode loop
 * (component/coolchic.py:89-166, latent.py:18-187, armint.py:180-203, rangecoder.py:87-94
 * -> constriction RangeDecoder.decode), Upsampling.forward (core/upsampling.py:463-500),
 * Synthesis.forward (core/synthesis.py:272-294) and the final F.interpolate
 * (component/coolchic.py:187-192).  Returns CCD_OK if every job succeeded, else the first
 * failing job's status. */
int ccd_decode_many(CcdContext *ctx, CcdJob *jobs, int n_jobs, void *cuda_stream);

/* Convenience: single job. */
int ccd_decode_coolchic(CcdContext *ctx, const CcdCoolChicDesc *desc, const uint8_t *nn_bytes,
                        size_t nn_nbytes, const uint8_t *latent_bytes, size_t latent_nbytes,
                        float *d_out, int8_t *d_latents, void *cuda_stream);

/* Stage entry point (used by tests / tools; same semantics as the entropy stage above). */
int ccd_decode_latents(CcdContext *ctx, const CcdCoolChicDesc *desc, const int64_t *nn_ints,
                       const uint8_t *latent_bytes, size_t latent_nbytes, int8_t *d_latents,
                       void *cuda_stream);

/* Range ENcoder on the device: the mode="encode" branch of the same reference functions
 * (component/coolchic.py:152-170,194-195, latent.py:166-170, rangecoder.py:46-78 ->
 * constriction RangeEncoder.encode / get_compressed).  mode 1: encode the latents found in
 * d_latents (decode order);  mode 2: DRAW the latents from the stream's own ARM (seeded
 * splitmix64, one 24-bit quantile per symbol), store them in d_latents and encode them --
 * used to fabricate self-consistent synthetic streams (SURVEY 8d).  Output: little-endian
 * u32 words in d_out_words (device), count in *n_words_out.  A symbol costs at most
 * 24 - log2(1 - 2^-8) < 24.0057 bits, so out_cap_words = ceil(n * 24.0057 / 32) + 3 always
 * suffices.  Mode 1 refuses a latent outside [-64, 63] with CCD_ERR_ARG, the message naming
 * the smallest such decode-order index. */
int ccd_encode_latents(CcdContext *ctx, const CcdCoolChicDesc *desc, const int64_t *nn_ints, int mode,
                       uint64_t seed, int8_t *d_latents, uint32_t *d_out_words, int64_t out_cap_words,
                       int64_t *n_words_out, int32_t *slow_path_count_out, void *cuda_stream);

/* The float tail of ccd_decode_many (upsampling cascade, synthesis, final resize and the optional frame tail) on
 * latents the caller supplies: d_out (and d_out_u, d_out_v with finish_bitdepth / finish_type, as in CcdJob) receives
 * exactly what ccd_decode_many writes for a stream whose decoded latents are d_latents, except that every grid g with
 * bit g of zero_grids set (g = 0: the finest) is read as all zeros.  nn_ints: the host NN integers (ccd_decode_nn).
 * d_latents: int8 in decode order, as CcdJob.d_latents receives them; read only.  A mask bit at or above n_grids, or
 * on a hyperlatent grid (those only feed the entropy model), makes the job CCD_ERR_ARG. */
typedef struct CcdSynthJob {
    const CcdCoolChicDesc *desc;
    const int64_t *nn_ints;
    const int8_t *d_latents;
    uint32_t zero_grids;
    float *d_out;
    int32_t finish_bitdepth, finish_type;
    float *d_out_u, *d_out_v;
    int32_t status;
} CcdSynthJob;

/* All jobs share the batched launches, one per cascade level and one per synthesis group, as in a decode; jobs outside
 * the batched path make their own launches.  No entropy launch.  One host->device and one device->host copy;
 * synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_synthesize_many(CcdContext *ctx, CcdSynthJob *jobs, int n_jobs, void *cuda_stream);

/* Rate analysis of decoded latents: the information content of every latent symbol under the model the
 * range coder used -- the ARM + IFCE evaluated exactly as decoding does, (mu_idx, sc_idx) clamped like
 * latent.py:165 / rangecoder.py:89-91, freq = left(s+1) - left(s) of constriction's leaky quantised Laplace
 * on the 2^24 scale (an integer in [1, 2^24]), bits = 24 - log2(freq).  This is not the encoder's training
 * rate proxy.  Inputs: desc, the host NN integers (ccd_decode_nn) and d_latents in decode order (what
 * ccd_decode_many writes to CcdJob.d_latents).  Outputs: d_bits float32 [n_symbols] in decode order
 * (required); d_freq uint32 and d_mu_sc (mu_idx | sc_idx << 16) uint32, same layout (optional);
 * d_spatial float32 [img_h][img_w] (optional): the per-pixel map of training/test.py:217-235 -- every
 * grid's bits divided by fp32((H*W)/(h*w)), taken to the image size by nearest (F.interpolate index),
 * summed over grids in fp32, finest grid first, starting from 0; grid_bits (out): f64 sum per grid
 * (grid 0 = finest), a fixed-order reduction (the same value on every run).  A latent outside [-64, 63]
 * makes the job CCD_ERR_ARG with bad_index = its decode-order index (else -1). */
typedef struct CcdRateJob {
    const CcdCoolChicDesc *desc;
    const int64_t *nn_ints;
    const int8_t *d_latents;
    float *d_bits;
    uint32_t *d_freq;
    uint32_t *d_mu_sc;
    float *d_spatial;
    double grid_bits[CCD_MAX_GRIDS];
    int64_t bad_index;
    int32_t status;
} CcdRateJob;

/* All jobs in ONE kernel launch (plus one for the spatial maps, if any job asks for one).  Synchronous
 * like ccd_decode_many.  Returns CCD_OK or the first failing job's status. */
int ccd_latent_rate(CcdContext *ctx, CcdRateJob *jobs, int n_jobs, void *cuda_stream);

/* Entropy-model analysis (DESIGN §4.10): the rate of ccd_latent_rate under the coder's model with some ARM inputs read
 * as 0, the model's own convention for a neighbour outside the grid and for a grid without IFCE input.  The first
 * operation on an ARM or IFCE input is linear, so an input read as 0 is its row of the first layer's (and the
 * stabiliser's) fixed-point weights set to 0; the library edits the weights on the host, and the edited model takes the
 * fast or the generic kernel by the decoder's own rule.
 *   zero_ctx:        bit t: spatial input t (the neighbour of priority t, core/arm.py:496-562) read as 0;
 *   zero_ifce_out:   bit c: IFCE feature c (ARM input n_ctx + c) read as 0;
 *   zero_ifce_grids: bit g (g = 0: the finest grid): latent grid g read as 0 wherever it is an IFCE input (channel c of
 *                    grid h reads grid h + 1 + c).
 * edits[i] applies to jobs[i]; edits == NULL edits nothing.  An all-zero edit gives exactly ccd_latent_rate's results.
 * CCD_ERR_ARG, before any launch: a zero_ctx bit >= n_ctx, a zero_ifce_out bit >= n_ifce_out, any IFCE bit in a model
 * without IFCE (flag_ifce 0), a zero_ifce_grids bit >= n_grids. */
typedef struct CcdModelEdit {
    uint64_t zero_ctx;
    uint32_t zero_ifce_out;
    uint32_t zero_ifce_grids;
} CcdModelEdit;
int ccd_latent_rate_edited(CcdContext *ctx, CcdRateJob *jobs, const CcdModelEdit *edits, int n_jobs, void *cuda_stream);

/* Scale-calibration sweep and static histogram of decoded latents (DESIGN §4.10), from the (mu_idx, sc_idx) the coder
 * used (d_mu_sc, as ccd_latent_rate writes it).  For each offset k < n_offsets, bits[g][k] (out) is the f64 sum over
 * grid g (0 = finest) of 24 - log2(freq) with sc_idx' = clamp(sc_idx + sc_offset[k], 0, 2560) and mu_idx unchanged:
 * the scale times exp(sc_offset[k] / 256).  The interval is ccd_latent_rate's (the table window, else the exact f64
 * model).  hist[g][s + 64] (out): the count of symbol s in grid g.  Sums are f64 partials per tile and offset added in
 * tile order, the histograms integer counts: the same on every run.  CCD_ERR_ARG before any launch: n_offsets outside
 * 1 .. 32, an offset outside [-2560, 2560]; after the launch, with bad_index = the smallest decode-order index of such a
 * symbol (else -1): a latent outside [-64, 63], a mu_idx above 32767 or an sc_idx above 2560. */
#define CCD_SWEEP_MAX_OFFSETS 32
typedef struct CcdSweepJob {
    const CcdCoolChicDesc *desc;
    const int8_t *d_latents;
    const uint32_t *d_mu_sc;
    int32_t n_offsets;
    int32_t sc_offset[CCD_SWEEP_MAX_OFFSETS];
    double bits[CCD_MAX_GRIDS][CCD_SWEEP_MAX_OFFSETS];
    uint64_t hist[CCD_MAX_GRIDS][128];
    int64_t bad_index;
    int32_t status;
} CcdSweepJob;

/* All jobs in ONE kernel launch; one copy each way; synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_rate_sweep(CcdContext *ctx, CcdSweepJob *jobs, int n_jobs, void *cuda_stream);

/* Candidate pricing for lossless model tuning (DESIGN §4.11): ccd_latent_rate's per-grid bits of one Cool-chic's decoded
 * latents under its model and under k candidate models, each of which adds delta to ONE transmitted ARM or IFCE integer
 * (nn_index into the ccd_decode_nn order: an ARM weight or bias, stabiliser included, or an IFCE weight or bias).
 * bits_out[c * n_grids + g] (out, grid 0 = finest): c = 0 the model itself, c = 1 + j candidate j; each equals, bit for
 * bit, ccd_latent_rate's grid_bits on the edited integers.  fast_out[c] (out, may be NULL): 1 if that model takes the
 * fast entropy kernel by the decoder's rule (arm_fits_f64 and the IFCE bound), else 0.  One kernel launch, one copy each
 * way, synchronous.  CCD_ERR_ARG, before any launch: k outside 1 .. CCD_CAND_MAX, an index outside the ARM and IFCE
 * integers, a delta of 0; after the launch: a latent outside [-64, 63]. */
#define CCD_CAND_MAX 64
typedef struct CcdCandidate {
    int32_t nn_index;
    int32_t delta;
} CcdCandidate;
int ccd_rate_candidates(CcdContext *ctx, const CcdCoolChicDesc *desc, const int64_t *nn_ints, const int8_t *d_latents,
                        const CcdCandidate *cands, int k, double *bits_out, int32_t *fast_out, void *cuda_stream);

/* Tail of decode_frame for every frame type (bitstream/decode.py:191-206 with
 * io/format/yuv.py:239-256,274-300): round to the 2^b-1 grid -> (444->420 2x2 average of
 * U,V) -> clamp [0,1] -> round again.  data_type: 0 rgb, 1 yuv420, 2 yuv444.
 * d_in [3][H][W];  rgb/444: d_out_a [3][H][W];  420: d_out_a=y [H][W], d_out_b=u, d_out_c=v
 * [H/2][W/2]. */
int ccd_finish_frame(CcdContext *ctx, const float *d_in, int h, int w, int bitdepth, int data_type,
                     float *d_out_a, float *d_out_b, float *d_out_c, void *cuda_stream);

/* One P/B frame (bitstream/decode.py:156-206: apply_global_translation globalmotion.py:151-160, Warper.forward
 * warp.py:294-397 in its training branch, alpha/beta blending, residue, frame tail).  d_residue [n_res_ch][H][W],
 * d_motion [n_mot_ch][H][W]: raw synthesis outputs, channel counts checked (P: 4 / 2, B: 5 / 4; the reference raises a
 * shape error otherwise).  ref0, ref1 (ignored for P): planes in the frame's layout -- frame_data_type 1 (yuv420):
 * y [H][W], u, v [H/2][W/2], read through convert_420_to_444 (io/format/yuv.py:303-316) folded into the gather index;
 * else three [H][W] planes.  bitdepth 1 .. 16: the finished frame; 0: the pre-rounding frame, three [H][W] planes
 * (4:4:4 references only).  global_flow: (x, y) per reference.  warp_filter_size 2 / 4: grid_sample bilinear / bicubic
 * (border, align_corners; frames of at least 2x2); 6 .. 14 even: windowed sinc (14: the largest value of the 4-bit
 * header field, header/header.py:217). */
typedef struct CcdInterFrame {
    const float *d_residue;
    int32_t n_res_ch;
    const float *d_motion;
    int32_t n_mot_ch;
    const float *ref0[3], *ref1[3];
    int32_t frame_data_type, bitdepth, h, w, is_b;
    int32_t global_flow[4];
    int32_t warp_filter_size;
} CcdInterFrame;

/* The whole reconstruction in ONE kernel; out_planes in the layout of the references. */
int ccd_reconstruct_frame(CcdContext *ctx, const CcdInterFrame *frame, float *const out_planes[3], void *cuda_stream);

/* Output packing on the device (io/format/yuv.py:150-162, ppm.py:160-203, png.py:44-62): finished
 * planes (values on the k / (2^b - 1) grid) -> integer samples round(x * (2^b - 1)), uint8 when
 * sample_bytes == 1, little-endian uint16 when 2.  interleaved == 0: the three planes one after the
 * other (planar YUV file order; chroma planes [H >> cs][W >> cs], cs = 1 for yuv420);
 * interleaved == 1 (cs must be 0): pixel-interleaved [H][W][3] (PPM / PNG order).  d_out holds
 * sample_bytes * (H*W + 2 * (H>>cs) * (W>>cs)) bytes. */
int ccd_pack_frame(CcdContext *ctx, const float *const planes[3], int h, int w, int chroma_shift,
                   int bitdepth, int sample_bytes, int interleaved, void *d_out, void *cuda_stream);

/* The same conversion for n samples that already lie in output order -- the planes of a BATCH of finished
 * planar frames stored one after the other (what ccd_decode_many writes when the caller hands it slices
 * of one buffer): one launch and one device-to-host copy for the whole batch instead of one per frame. */
int ccd_pack_samples(CcdContext *ctx, const float *d_samples, size_t n, int bitdepth, int sample_bytes,
                     void *d_out, void *cuda_stream);

/* Distortion of finished frames against their source (training/loss.py:88-118 restated on integers): every decoded
 * sample x goes back to kd = rint(x * M), M = 2^bitdepth - 1, and d = kd - ks with ks the source sample.
 * d_planes: the finished frame in FrameData layout (three [H][W] planes; chroma_shift 1: planes 1, 2 are
 * [H/2][W/2], H and W even).  d_src: the source samples as read from the file, uint8 when bitdepth <= 8 else
 * native-endian uint16; src_layout 0: planar (Y, U, V one after the other), 1: [H][W][3] (chroma_shift 0 only).
 * d_map (optional): float32 [H][W], fp32(sum_c d_c^2) / fp32(M^2), 4:2:0 chroma read at (y >> 1, x >> 1).
 * Outputs: sse[c] = sum of d^2 over plane c (exact), max_abs[c] = max |d|.  A decoded value off the k / M grid
 * (|x * M - kd| > 1/16, or x outside [0, 1]) makes the job CCD_ERR_ARG with bad_index = the smallest such
 * sample's planar index (plane after plane, each row-major; else -1). */
typedef struct CcdDistJob {
    const float *d_planes[3];
    const void *d_src;
    int32_t h, w, chroma_shift, bitdepth, src_layout;
    float *d_map;
    uint64_t sse[3];
    uint32_t max_abs[3];
    int64_t bad_index;
    int32_t status;
} CcdDistJob;

/* All jobs in ONE kernel launch; synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_frame_distortion(CcdContext *ctx, CcdDistJob *jobs, int n_jobs, void *cuda_stream);

/* MS-SSIM of finished frames against their source (Wang, Simoncelli and Bovik 2003; DESIGN §4.6), from the same
 * integers as ccd_frame_distortion: kd = rint(x * M) against ks, data range M, C1 = (0.01 M)^2, C2 = (0.03 M)^2.
 * Inputs as for CcdDistJob.  Each plane at its own resolution: scale 0 is the plane, scale j + 1 the 2 x 2 average
 * of scale j (floor sizes); an 11-tap Gaussian window (sigma 1.5), "valid" filtering.  Every plane needs both
 * sides >= 176 (five scales of at least 11 samples), else CCD_ERR_ARG.
 * d_map[c] (optional): float32 [h_c - 10][w_c - 10], the scale-0 SSIM map (l * cs) of plane c.
 * Outputs: cs[c][j] = mean of cs, ssim[c][j] = mean of l * cs over plane c at scale j (f64 partials per tile added
 * in tile order: the same on every run).  An off-grid decoded value is reported as by ccd_frame_distortion. */
typedef struct CcdSsimJob {
    const float *d_planes[3];
    const void *d_src;
    int32_t h, w, chroma_shift, bitdepth, src_layout;
    float *d_map[3];
    double cs[3][5];
    double ssim[3][5];
    int64_t bad_index;
    int32_t status;
} CcdSsimJob;

/* All jobs in five kernel launches, one per scale; synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_frame_ssim(CcdContext *ctx, CcdSsimJob *jobs, int n_jobs, void *cuda_stream);

/* Multi-scale pixel-domain VIF of finished frames against their source (Sheikh and Bovik 2006, the LIVE vifp_mscale;
 * DESIGN §4.12).  Inputs as for CcdDistJob; the source is the reference image, the decoded frame the distorted one,
 * both in 8-bit units v = k * 255 / M (f64), so the model's noise variance 2 means the same at every bit depth.  Each
 * plane at its own resolution.  Scale s = 0..3 uses an N_s = 2^(4 - s) + 1 tap Gaussian window (sigma N_s / 5),
 * "valid"; scale s >= 1 is scale s - 1 filtered with scale s's window and decimated to its even rows and columns.
 * Every plane needs both sides >= 41 (a valid output at scale 3), else CCD_ERR_ARG before any launch.
 * Outputs: num[c][s], den[c][s] = the sums over plane c at scale s of log10(1 + g^2 sigma_ref^2 / (sv^2 + 2)) and of
 * log10(1 + sigma_ref^2 / 2) (f64 partials per tile added in tile order: the same on every run); the plane's VIF is
 * sum_s num / sum_s den.  An off-grid decoded value is reported as by ccd_frame_distortion. */
typedef struct CcdVifJob {
    const float *d_planes[3];
    const void *d_src;
    int32_t h, w, chroma_shift, bitdepth, src_layout;
    double num[3][4];
    double den[3][4];
    int64_t bad_index;
    int32_t status;
} CcdVifJob;

/* All jobs in four kernel launches, one per scale; synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_frame_vif(CcdContext *ctx, CcdVifJob *jobs, int n_jobs, void *cuda_stream);

/* PSNR-HVS-M and PSNR-HVS of finished frames against their source (Ponomarenko et al. 2007; DESIGN §4.13).  Inputs as
 * for CcdDistJob; both images in 8-bit units v = k * 255 / M (f64).  Each plane at its own resolution, cut into the
 * non-overlapping 8 x 8 blocks that lie wholly inside it (the other samples are read only for the off-grid check);
 * per block the orthonormal 2-D DCT-II of both images, the contrast masking of the larger of the two blocks' masks,
 * and the CSF-weighted squared coefficient errors.  Every plane needs both sides >= 8, else CCD_ERR_ARG before any
 * launch.
 * d_map[c] (optional): float32 [h_c >> 3][w_c >> 3], each block's S_hvs_m / 64 / 255^2.
 * Outputs: s_hvs_m[c], s_hvs[c] = the sums over plane c's blocks of the masked and unmasked weighted squared errors
 * (f64 partials per tile added in tile order: the same on every run); with N_c = 64 blocks, the plane's PSNR-HVS-M is
 * -10 log10(s_hvs_m / N_c / 255^2).  An off-grid decoded value is reported as by ccd_frame_distortion. */
typedef struct CcdHvsJob {
    const float *d_planes[3];
    const void *d_src;
    int32_t h, w, chroma_shift, bitdepth, src_layout;
    float *d_map[3];
    double s_hvs_m[3];
    double s_hvs[3];
    int64_t bad_index;
    int32_t status;
} CcdHvsJob;

/* All jobs in ONE kernel launch; synchronous.  Returns CCD_OK or the first failing job's status. */
int ccd_frame_hvs(CcdContext *ctx, CcdHvsJob *jobs, int n_jobs, void *cuda_stream);

/* Statistics of a P/B frame's prediction (training/test.py:169-199), with the fp32 operations of the reconstruction
 * (bitdepth >= 1: the source scale): pred (beta * p0 + (1 - beta) * p1 for B), alpha, beta.  d_src (optional): source
 * samples as for ccd_frame_distortion (src_layout 1 not for yuv420); orig = ks / M, 4:2:0 chroma read at >> 1,
 * dummy = ((0 + r0) + r1) / n_refs.  Optional maps: d_alpha, d_beta [H][W], d_pred [3][H][W].  sums (out): sum of
 * alpha, of beta (0 for P) and, with a source (else 0), of fp32((pred - orig)^2) and fp32((dummy - orig)^2) over the
 * 3 H W samples: f64 partials per CTA added in tile order, the same on every run.  One launch; synchronous. */
typedef struct CcdInterStats {
    const void *d_src;
    int32_t src_layout;
    float *d_alpha, *d_beta, *d_pred;
    double sums[4];
} CcdInterStats;
int ccd_inter_stats(CcdContext *ctx, const CcdInterFrame *frame, CcdInterStats *stats, void *cuda_stream);

/* Motion analysis of a P/B frame (DESIGN §4.9): what the motion, each reference and the residue buy.  A variant is the
 * finished frame of ccd_reconstruct_frame with one change to its inputs (bitdepth >= 1):
 *   0 decoded          none
 *   1 no_local_motion  every motion channel := 0, global flow kept
 *   2 no_motion        every motion channel := 0 and global flow := 0
 *   3 ref0_only        residue channel 4 := +0.5 (beta = 1), B only
 *   4 ref1_only        residue channel 4 := -0.5 (beta = 0), B only
 *   5 no_residue       residue channels 0..2 := 0
 *   6 no_prediction    residue channel 3 := -0.5 (alpha = 0)
 * sse[v][c] (out): sum of d^2 over plane c of variant v, d = rint(x * M) - ks as ccd_frame_distortion computes it
 * (exact; 0 for variants 3, 4 of a P frame).  d_src and src_layout as for CcdInterStats, the source is required.
 * Per reference r (ref 1: B only, else 0), over the H W luma pixels, with (fx, fy) motion channels 2r, 2r + 1 and (gx, gy)
 * its global flow: flow_sum[r] = sums of fx + gx, fy + gy and sqrt(fx^2 + fy^2), all in f64 (f64 partials per CTA
 * added in tile order, the same on every run); flow_max[r] = max sqrt(fx^2 + fy^2); outside[r] = pixels whose sample
 * position x + gx + fx or y + gy + fy (f64) lies outside [0, W - 1] or [0, H - 1].  d_flow[r] (optional): [2][H][W]
 * fp32 fx + gx, fy + gy.  A non-finite flow makes the call CCD_ERR_ARG with bad_index = the smallest such pixel
 * (row-major; else -1).  One launch; synchronous. */
#define CCD_INTER_VARIANTS 7
typedef struct CcdInterAnalysis {
    const void *d_src;
    int32_t src_layout;
    float *d_flow[2];
    uint64_t sse[CCD_INTER_VARIANTS][3];
    double flow_sum[2][3];
    double flow_max[2];
    uint64_t outside[2];
    int64_t bad_index;
    int32_t status;
} CcdInterAnalysis;
int ccd_inter_analysis(CcdContext *ctx, const CcdInterFrame *frame, CcdInterAnalysis *analysis, void *cuda_stream);

/* Device-side evaluation of the quantised-Laplace left cumulative for testing the f64
 * exp() agreement with the host (SURVEY Appendix C.3): for sc in [sc_lo, sc_hi) and every
 * numerator index n in [0, 32641) (|d| = n/256), writes to host arrays
 * out_lo[(sc-sc_lo)*32641+n] = trunc(FW * 0.5*exp(-|d|/b)) and
 * out_hi[...]                = trunc(FW * (1 - 0.5*exp(-|d|/b))). */
int ccd_debug_laplace_domain(CcdContext *ctx, int sc_lo, int sc_hi, uint32_t *out_lo,
                             uint32_t *out_hi);

/* The context's cumulative table, as the entropy decoder and the rate pass read it: for sc in
 * [sc_lo, sc_hi), f < 256, t < 32, writes to the host array
 * out[((sc-sc_lo)*256+f)*32+t] = trunc(FW * cdf(n/256)), n = 256 t - f - 3584 (window entry t of a
 * symbol whose mu_idx has (mu_idx + 128) & 255 = f). */
int ccd_debug_cdf_table(CcdContext *ctx, int sc_lo, int sc_hi, uint32_t *out);

/* Device-side evaluation of the canonical elementary functions (csrc/ccd_detmath.h), for testing them
 * against the host's copy bit for bit: y[i] = sin / cos / log (fn 0 / 1 / 2) of x[i], host arrays of n
 * doubles.  One launch; synchronous. */
int ccd_debug_detmath(CcdContext *ctx, int fn, const double *x, double *y, size_t n);

/* The taps of the windowed-sinc warp as the P/B kernels form them (warp.py:226-268), for taps = N in
 * {6, 8, 10, 12, 14}: c[N i + k] = tap k at the fractional offset s[i], host arrays.  Any other N is
 * CCD_ERR_ARG.  One launch; synchronous. */
int ccd_debug_sinc_coeffs(CcdContext *ctx, int taps, const float *s, float *c, size_t n);

/* Samples [first, first + n) of the common-randomness generator (noise.py:18-34) as the synthesis draws
 * them, before any resize, into the host array out.  One launch; synchronous. */
int ccd_debug_cr_noise(CcdContext *ctx, uint64_t first, size_t n, float *out);

/* Number of CUDA kernels this library has launched since it was loaded. */
uint64_t ccd_debug_launch_count(void);

/* Tuning knob: which of warps 0..14 of the entropy CTA act as ARM producers (bit i = warp i;
 * warp 14 is the coder's helper, warp 15 the range coder).  Default 0x3777: warps 3, 7, 11 stay idle so
 * that the coder owns scheduler partition 3. */
int ccd_debug_set_producer_mask(CcdContext *ctx, uint32_t mask);

/* Entropy-kernel status words of the last job of the last call: [0] error, [1] words consumed,
 * [2] slow-path symbols (outside the 31-symbol window), [3] words emitted (encode modes),
 * [4..15] cycle / event counters when the library is built with -DCCD_PROFILE (else 0; layout in
 * csrc/ccd_entropy.cu). */
int ccd_debug_last_status(const CcdContext *ctx, int32_t st[16]);

/* Shared-memory plan of the entropy kernel for one Cool-chic, computed on the host (no device needed) from its
 * descriptor and network integers (ccd_nn_count of them): out[0] window-ring slots, out[1] row-ring rows, out[2]
 * bytes of dynamic shared memory.  The out values are written even when the stream cannot be decoded, which is
 * then reported with CCD_ERR_UNSUPPORTED, as decoding would report it. */
int ccd_debug_entropy_plan(const CcdCoolChicDesc *desc, const int64_t *nn_ints, int64_t out[3]);

/* Timing of the last ccd_decode_many call on this context, measured with CUDA events on the
 * launching stream: ms[0] entropy stage, ms[1] upsampling+synthesis, ms[2] host prep + H2D;
 * ms[3] = bytes uploaded host->device by that call (as a float). */
int ccd_last_timing(const CcdContext *ctx, float ms[4]);

#ifdef __cplusplus
}
#endif
#endif
