/* ccoracle.c -- CPU restatement of the Cool-chic 5.0.1 decode path (plain C, scalar).
 *
 * TEST INFRASTRUCTURE ONLY (see ccoracle.h).  Build: `make -C oracle` -> oracle/_build/.
 * Compiled with -fwrapv -ffp-contract=off: int64 wraps like torch.int64, and no implicit
 * FMA contraction -- every fused multiply-add below is an explicit fmaf().
 *
 * Canonical fp32 order (the reference itself is not bit-stable across thread counts,
 * SURVEY F7): each convolution output is  acc = init; for ci, for ky, for kx:
 * acc = fmaf(w, x, acc)  with init = bias (synthesis) or 0 (upsampling).  The CUDA kernels
 * of the product replicate exactly this order, so GPU == oracle bit for bit, and both are
 * within 1e-5 of the PyTorch reference.
 */
#include "ccoracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "detmath.h"

static const uint32_t k_scale_bits[2561] = {
#include "scale_table.inc"
};

static inline float scale_from_index(int idx) {
    float f;
    memcpy(&f, &k_scale_bits[idx], 4);
    return f;
}

int cco_sizeof_desc(void) { return (int)sizeof(CcoDesc); }

/* The float tail is parallelised over output rows with OpenMP (results are independent of
 * the thread count: every output keeps its own fixed summation order); the entropy stage
 * of one stream is inherently serial.  cco_set_threads(0) = all cores. */
#ifdef _OPENMP
#include <omp.h>
int cco_set_threads(int n) {
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
}
#else
int cco_set_threads(int n) { (void)n; return 1; }
#endif

/* ------------------------------------------------------------------------------------ */
/* Context pattern: reference core/arm.py:496-562 (priority order over the 9x9 causal
 * mask; first n_ctx entries are used).  (dy, dx) relative to the coded pixel.          */
static const int8_t k_ctx_dy[40] = {0,  -1, -1, -1, 0,  -2, -3, 0,  -1, -2, -2, -1, -2, -1,
                                    -2, -3, 0,  -1, -2, -2, -3, -3, -3, -4, -1, -4, -1, -2,
                                    -3, -3, -4, -4, -2, -3, -3, -4, -4, -4, -4, -4};
static const int8_t k_ctx_dx[40] = {-1, 0,  -1, 1, -2, 0,  0,  -3, -2, 1,  -1, 2,  -2, -3,
                                    2,  1,  -4, 3, -3, 3,  -1, -2, 2,  0,  -4, -1, 4,  4,
                                    -3, 3,  -2, 1, -4, -4, 4,  -3, 2,  3,  -4, 4};
#define ARM_MASK 9
#define ARM_PAD 4
#define WAVE_STRIDE (ARM_MASK + 1)

/* ------------------------------------------------------------------------------------ */
/* NN parameter layout: neuralnet.py:120-148 (order arm, ifce, upsampling, synthesis;
 * within a module all weights then all biases; registration orders from arm.py:176-195,
 * arm.py:336-350, upsampling.py:428-437 (+ parametrize), synthesis.py:197-241).          */
typedef struct {
    int dim;                  /* ARM width = n_ctx + n_ifce_out */
    int n_arm_lin;            /* hidden + 1 */
    int64_t off_arm_w[9], off_arm_b[9]; /* per linear layer; index n_arm_lin = stabiliser */
    int n_ifce;               /* number of IFCE arms */
    int ifce_grid[CCO_MAX_GRIDS];
    int64_t off_ifce_w[CCO_MAX_GRIDS], off_ifce_b[CCO_MAX_GRIDS];
    int kt_par, kc_par;       /* transmitted taps per kernel */
    int64_t off_ups_tw, off_ups_cw, off_ups_tb, off_ups_cb;
    int syn_c_out, syn_stab_in;
    int64_t off_syn_ot_w, off_syn_st_w, off_syn_w[CCO_MAX_SYN];
    int64_t off_syn_ot_b, off_syn_st_b, off_syn_b[CCO_MAX_SYN];
    int64_t counts[8];
    int64_t total;
} NNLayout;

static int nn_layout(const CcoDesc *d, NNLayout *L) {
    memset(L, 0, sizeof(*L));
    if (d->n_grids < 1 || d->n_grids > CCO_MAX_GRIDS) return CCO_ERR_ARG;
    if (d->n_syn_layers < 1 || d->n_syn_layers > CCO_MAX_SYN) return CCO_ERR_ARG;
    if (d->arm_hidden < 0 || d->arm_hidden > 7) return CCO_ERR_ARG;
    if (d->n_ctx < 0 || d->n_ctx > 40) return CCO_ERR_ARG;
    int64_t p = 0;
    int dim = d->n_ctx + d->n_ifce_out;
    L->dim = dim;
    L->n_arm_lin = d->arm_hidden + 1;
    /* arm weights */
    for (int l = 0; l < L->n_arm_lin; l++) {
        int out = (l == d->arm_hidden) ? 2 : dim;
        L->off_arm_w[l] = p;
        p += (int64_t)out * dim;
    }
    if (d->arm_stab) {
        L->off_arm_w[L->n_arm_lin] = p;
        p += 2 * dim;
    }
    L->counts[0] = p;
    int64_t q = p;
    for (int l = 0; l < L->n_arm_lin; l++) {
        int out = (l == d->arm_hidden) ? 2 : dim;
        L->off_arm_b[l] = p;
        p += out;
    }
    if (d->arm_stab) {
        L->off_arm_b[L->n_arm_lin] = p;
        p += 2;
    }
    L->counts[1] = p - q;
    /* ifce */
    q = p;
    if (d->flag_ifce) {
        for (int g = 0; g < d->n_grids; g++) {
            if (d->grid_ifce_in[g] > 0) {
                L->ifce_grid[L->n_ifce] = g;
                L->off_ifce_w[L->n_ifce] = p;
                p += (int64_t)d->n_ifce_out * d->grid_ifce_in[g];
                L->n_ifce++;
            }
        }
    }
    L->counts[2] = p - q;
    q = p;
    for (int j = 0; j < L->n_ifce; j++) {
        L->off_ifce_b[j] = p;
        p += d->n_ifce_out;
    }
    L->counts[3] = p - q;
    /* upsampling */
    L->kt_par = (d->ups_k + 1) / 2;
    L->kc_par = (d->ups_pre_k + 1) / 2;
    q = p;
    L->off_ups_tw = p;
    p += (int64_t)d->n_ups * L->kt_par;
    L->off_ups_cw = p;
    p += (int64_t)d->n_ups * L->kc_par;
    L->counts[4] = p - q;
    q = p;
    L->off_ups_tb = p;
    p += d->n_ups;
    L->off_ups_cb = p;
    p += d->n_ups;
    L->counts[5] = p - q;
    /* synthesis */
    int C = d->syn_out[d->n_syn_layers - 1];
    L->syn_c_out = C;
    L->syn_stab_in = d->common_randomness ? d->syn_in / 2 : d->syn_in;
    q = p;
    L->off_syn_ot_w = p;
    p += (int64_t)C * C;
    if (d->syn_stab) {
        L->off_syn_st_w = p;
        p += (int64_t)C * L->syn_stab_in;
    }
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        L->off_syn_w[l] = p;
        p += (int64_t)d->syn_out[l] * in_ft * d->syn_k[l] * d->syn_k[l];
        in_ft = d->syn_out[l];
    }
    L->counts[6] = p - q;
    q = p;
    L->off_syn_ot_b = p;
    p += C;
    if (d->syn_stab) {
        L->off_syn_st_b = p;
        p += C;
    }
    for (int l = 0; l < d->n_syn_layers; l++) {
        L->off_syn_b[l] = p;
        p += d->syn_out[l];
    }
    L->counts[7] = p - q;
    L->total = p;
    return CCO_OK;
}

int64_t cco_nn_counts(const CcoDesc *d, int64_t counts[8]) {
    NNLayout L;
    int rc = nn_layout(d, &L);
    if (rc) return rc;
    if (counts) memcpy(counts, L.counts, sizeof(L.counts));
    return L.total;
}

/* ------------------------------------------------------------------------------------ */
/* exp-Golomb: neuralnet/expgolomb.py:74-130 (decode), :15-71 (encode).  MSB-first bits,
 * payload is prefixed with nn_n_bit_pad padding bits.                                    */
typedef struct {
    const uint8_t *p;
    size_t nbits, pos;
} BitRd;
static inline int rd_bit(BitRd *b) {
    if (b->pos >= b->nbits) return -1;
    int v = (b->p[b->pos >> 3] >> (7 - (b->pos & 7))) & 1;
    b->pos++;
    return v;
}

int64_t cco_decode_nn(const CcoDesc *d, const uint8_t *bytes, size_t nbytes, int64_t *out,
                      size_t cap) {
    NNLayout L;
    int rc = nn_layout(d, &L);
    if (rc) return rc;
    if ((size_t)L.total > cap) return CCO_ERR_ARG;
    BitRd br = {bytes, nbytes * 8, (size_t)d->nn_n_bit_pad};
    int64_t n = 0;
    for (int m = 0; m < 8; m++) {
        int k = d->expgol[m];
        for (int64_t i = 0; i < L.counts[m]; i++) {
            int nread = 1, bit;
            while ((bit = rd_bit(&br)) == 0) nread++;
            if (bit < 0) return CCO_ERR_NN_TRUNCATED;
            if (nread > 62) return CCO_ERR_NN_TRUNCATED;
            uint64_t val = 1;
            for (int j = 1; j < nread; j++) {
                bit = rd_bit(&br);
                if (bit < 0) return CCO_ERR_NN_TRUNCATED;
                val = (val << 1) | (uint64_t)bit;
            }
            uint64_t quotient = val - 1, rem = 0;
            for (int j = 0; j < k; j++) {
                bit = rd_bit(&br);
                if (bit < 0) return CCO_ERR_NN_TRUNCATED;
                rem = (rem << 1) | (uint64_t)bit;
            }
            int64_t v = (int64_t)((quotient << k) + rem);
            out[n++] = (v & 1) ? (v + 1) / 2 : -(v / 2);
        }
    }
    return n;
}

int64_t cco_encode_nn(const CcoDesc *d, const int64_t *ints, size_t n, uint8_t *out, size_t cap,
                      int32_t *n_pad) {
    NNLayout L;
    int rc = nn_layout(d, &L);
    if (rc) return rc;
    if ((int64_t)n != L.total) return CCO_ERR_ARG;
    /* first pass: count bits */
    size_t nbits = 0;
    for (int pass = 0; pass < 2; pass++) {
        size_t pos = 0;
        if (pass == 1) {
            size_t pad = (8 - nbits % 8) % 8;
            if ((nbits + pad) / 8 > cap) return CCO_ERR_ARG;
            memset(out, 0, (nbits + pad) / 8);
            *n_pad = (int32_t)pad;
            pos = pad;
        }
        int64_t idx = 0;
        for (int m = 0; m < 8; m++) {
            int k = d->expgol[m];
            for (int64_t i = 0; i < L.counts[m]; i++, idx++) {
                int64_t x = ints[idx];
                uint64_t u = (x <= 0) ? (uint64_t)(-2 * x) : (uint64_t)(2 * x - 1);
                u += ((uint64_t)1 << k) - 1; /* order-0 code of u+1 with k leading zeros removed */
                uint64_t v = u + 1;
                int len = 64 - __builtin_clzll(v); /* bits of v */
                int total = 2 * len - 1 - k;       /* (len-1) zeros + len bits, minus k zeros */
                if (pass == 1) {
                    size_t start = pos + (size_t)(len - 1 - k);
                    for (int j = 0; j < len; j++)
                        if ((v >> (len - 1 - j)) & 1) out[(start + j) >> 3] |= (uint8_t)(0x80 >> ((start + j) & 7));
                }
                pos += (size_t)total;
            }
        }
        if (pass == 0) nbits = pos;
    }
    size_t pad = (8 - nbits % 8) % 8;
    return (int64_t)((nbits + pad) / 8);
}

/* ------------------------------------------------------------------------------------ */
/* Integer ARM parameters: armint.py:30-170.                                              */
typedef struct {
    int dim, n_lin;  /* n_lin linear layers in the trunk */
    int out_last;
    int64_t *W[8];   /* transposed: W[l][in*out_l + out] */
    int64_t *B[8];
    int64_t *Ws, *Bs; /* stabiliser [in*2+out], [2]; zeros if absent */
} ArmFP;

static void armfp_free(ArmFP *a) {
    for (int l = 0; l < 8; l++) {
        free(a->W[l]);
        free(a->B[l]);
    }
    free(a->Ws);
    free(a->Bs);
    memset(a, 0, sizeof(*a));
}

/* One module (main ARM or one IFCE arm). qw/qb point to the raw transmitted ints of each
 * linear layer ([out][in] row-major) -- armint.py:73-131. */
static int armfp_build(ArmFP *a, int dim, int n_hidden, int n_out, const int64_t *const *qw,
                       const int64_t *const *qb, const int64_t *qws, const int64_t *qbs, int s_w,
                       int s_b, int subtract_last, int n_inter_ft, int no_residual) {
    memset(a, 0, sizeof(*a));
    a->dim = dim;
    a->n_lin = n_hidden + 1;
    a->out_last = n_out;
    for (int l = 0; l < a->n_lin; l++) {
        int out = (l == n_hidden) ? n_out : dim;
        a->W[l] = (int64_t *)calloc((size_t)dim * out + 1, 8);
        a->B[l] = (int64_t *)calloc((size_t)out + 1, 8);
        if (!a->W[l] || !a->B[l]) return CCO_ERR_NOMEM;
        for (int o = 0; o < out; o++) {
            for (int i = 0; i < dim; i++) {
                int shift = 16 + s_w;
                int ifce_col = (n_inter_ft > 0 && l == 0 && i >= dim - n_inter_ft);
                if (ifce_col) shift -= 8;
                int64_t v = qw[l][(size_t)o * dim + i] * ((int64_t)1 << shift);
                if (out == dim && !no_residual && o == i) v += (int64_t)1 << (ifce_col ? 8 : 16);
                a->W[l][(size_t)i * out + o] = v;
            }
            int64_t qv = qb[l][o];
            if (l == n_hidden && subtract_last && o == 1) qv += -((int64_t)4 << (-s_b));
            a->B[l][o] = qv * ((int64_t)1 << (32 + s_b));
        }
    }
    a->Ws = (int64_t *)calloc((size_t)dim * n_out + 1, 8);
    a->Bs = (int64_t *)calloc((size_t)n_out + 1, 8);
    if (!a->Ws || !a->Bs) return CCO_ERR_NOMEM;
    if (qws) {
        for (int o = 0; o < n_out; o++) {
            for (int i = 0; i < dim; i++) {
                int shift = 16 + s_w;
                if (n_inter_ft > 0 && i >= dim - n_inter_ft) shift -= 8;
                a->Ws[(size_t)i * n_out + o] = qws[(size_t)o * dim + i] * ((int64_t)1 << shift);
            }
            a->Bs[o] = qbs[o] * ((int64_t)1 << (32 + s_b));
        }
    }
    return CCO_OK;
}

/* armint.py:180-203.  ctx: dim integers; out: out_last integers after >> output_shift. */
static void armfp_forward(const ArmFP *a, const int64_t *ctx, int64_t *out, int output_shift,
                          int64_t *stat_acc, int64_t *stat_hid) {
    int64_t x[80], y[80], stab[32];
    int dim = a->dim;
    for (int i = 0; i < dim; i++) x[i] = ctx[i] << 16;
    for (int o = 0; o < a->out_last; o++) {
        int64_t acc = a->Bs[o];
        for (int i = 0; i < dim; i++) acc += x[i] * a->Ws[(size_t)i * a->out_last + o];
        stab[o] = acc;
    }
    for (int l = 0; l < a->n_lin - 1; l++) {
        for (int o = 0; o < dim; o++) {
            int64_t acc = a->B[l][o];
            for (int i = 0; i < dim; i++) acc += x[i] * a->W[l][(size_t)i * dim + o];
            if (stat_acc) {
                int64_t m = acc < 0 ? -acc : acc;
                if (m > *stat_acc) *stat_acc = m;
            }
            if (acc < 0) acc = 0;
            y[o] = acc >> 16;
            if (stat_hid && y[o] > *stat_hid) *stat_hid = y[o];
        }
        memcpy(x, y, sizeof(int64_t) * (size_t)dim);
    }
    int l = a->n_lin - 1;
    for (int o = 0; o < a->out_last; o++) {
        int64_t acc = a->B[l][o];
        for (int i = 0; i < dim; i++) acc += x[i] * a->W[l][(size_t)i * a->out_last + o];
        acc += stab[o];
        if (stat_acc) {
            int64_t m = acc < 0 ? -acc : acc;
            if (m > *stat_acc) *stat_acc = m;
        }
        out[o] = acc >> output_shift;
    }
}

/* ------------------------------------------------------------------------------------ */
/* constriction 0.4.2 restated: QuantizedLaplace(-64, 63) leaky quantiser (f64) and the
 * queue RangeDecoder / RangeEncoder (u32 words, u64 state, 24-bit precision).
 * Call sites in the reference: rangecoder.py:30-34, 62, 82, 93.   SURVEY Appendix C.    */
#define RC_PREC 24
#define SYM_MIN (-64)
#define SYM_MAX 63
static const double k_free_weight = 16777215.0 - 127.0; /* (2^24-1) - (max-min) */

static inline uint32_t laplace_left(int s, double mu, double b) {
    if (s <= SYM_MIN) return 0;
    if (s > SYM_MAX) return 1u << RC_PREC;
    double x = (double)s - 0.5, c;
    if (x <= mu)
        c = 0.5 * exp((x - mu) / b);
    else
        c = 1.0 - 0.5 * exp((mu - x) / b);
    return (uint32_t)(k_free_weight * c) + (uint32_t)(s - SYM_MIN);
}
/* Host (libm) image of ccd_debug_laplace_domain: every |d| = n/256, n in [0, 32641), for the
 * scales [sc_lo, sc_hi): trunc(FW*0.5*exp(-|d|/b)) and trunc(FW*(1-0.5*exp(-|d|/b))). */
void cco_laplace_domain(int sc_lo, int sc_hi, uint32_t *lo, uint32_t *hi) {
    const int ND = 32641;
    for (int sc = sc_lo; sc < sc_hi; sc++) {
        double b = (double)scale_from_index(sc);
        for (int n = 0; n < ND; n++) {
            double d = (double)n * (1.0 / 256.0);
            size_t i = (size_t)(sc - sc_lo) * ND + (size_t)n;
            lo[i] = (uint32_t)(k_free_weight * (0.5 * exp(-d / b)));
            hi[i] = (n == 0) ? lo[i] : (uint32_t)(k_free_weight * (1.0 - 0.5 * exp(-d / b)));
        }
    }
}

uint32_t cco_laplace_left(int s, float mu, float scale) {
    return laplace_left(s, (double)mu, (double)scale);
}

typedef struct {
    const uint32_t *w;
    size_t n, pos;
    uint64_t lower, range, point;
} RcDec;

static inline uint32_t rc_next(RcDec *r) {
    uint32_t v = (r->pos < r->n) ? r->w[r->pos] : 0;
    r->pos++;
    return v;
}
static void rc_dec_init(RcDec *r, const uint32_t *w, size_t n) {
    r->w = w;
    r->n = n;
    r->pos = 0;
    r->lower = 0;
    r->range = ~(uint64_t)0;
    uint64_t hi = rc_next(r);
    r->point = (hi << 32) | rc_next(r);
}

/* find s with left(s) <= q < left(s+1); returns left and left(s+1) */
static inline int laplace_find(uint32_t q, double mu, double b, uint32_t *pl, uint32_t *pr) {
    int s = (int)lrint(mu);
    if (s < SYM_MIN) s = SYM_MIN;
    if (s > SYM_MAX) s = SYM_MAX;
    uint32_t l = laplace_left(s, mu, b);
    if (l > q) {
        uint32_t r;
        do {
            r = l;
            s--;
            l = laplace_left(s, mu, b);
        } while (l > q);
        *pl = l;
        *pr = r;
        return s;
    }
    uint32_t r = laplace_left(s + 1, mu, b);
    while (r <= q) {
        l = r;
        s++;
        r = laplace_left(s + 1, mu, b);
    }
    *pl = l;
    *pr = r;
    return s;
}

static inline int rc_decode(RcDec *r, double mu, double b, int *sym) {
    uint64_t scale = r->range >> RC_PREC;
    uint64_t q = (r->point - r->lower) / scale;
    if (q >= ((uint64_t)1 << RC_PREC)) return CCO_ERR_DESYNC;
    uint32_t l, rr;
    *sym = laplace_find((uint32_t)q, mu, b, &l, &rr);
    r->lower += scale * l;
    r->range = scale * (uint64_t)(rr - l);
    if (r->range < ((uint64_t)1 << 32)) {
        r->lower <<= 32;
        r->range <<= 32;
        r->point = (r->point << 32) | rc_next(r);
    }
    return CCO_OK;
}

void *cco_rc_dec_new(const uint32_t *words, size_t n) {
    RcDec *r = (RcDec *)malloc(sizeof(RcDec));
    if (r) rc_dec_init(r, words, n);
    return r;
}
void cco_rc_dec_free(void *h) { free(h); }
int cco_rc_decode_block(void *h, const float *mu, const float *scale, int n, int32_t *out) {
    RcDec *r = (RcDec *)h;
    for (int i = 0; i < n; i++) {
        int s;
        int rc = rc_decode(r, (double)mu[i], (double)scale[i], &s);
        if (rc) return rc;
        out[i] = s;
    }
    return CCO_OK;
}

typedef struct {
    uint32_t *w;
    size_t n, cap;
    uint64_t lower, range;
    uint64_t nsym;
    int oom;
} RcEnc;

static void rc_enc_push(RcEnc *e, uint32_t v) {
    if (e->n == e->cap) {
        size_t nc = e->cap ? e->cap * 2 : 1024;
        uint32_t *nw = (uint32_t *)realloc(e->w, nc * 4);
        if (!nw) {
            e->oom = 1;
            return;
        }
        e->w = nw;
        e->cap = nc;
    }
    e->w[e->n++] = v;
}
static void rc_enc_carry(RcEnc *e) {
    size_t i = e->n;
    while (i > 0) {
        i--;
        if (++e->w[i] != 0) break;
    }
}
static void rc_enc_init(RcEnc *e) {
    memset(e, 0, sizeof(*e));
    e->range = ~(uint64_t)0;
}
static void rc_encode(RcEnc *e, int s, double mu, double b) {
    uint32_t l = laplace_left(s, mu, b), r = laplace_left(s + 1, mu, b);
    uint64_t scale = e->range >> RC_PREC;
    uint64_t nl = e->lower + scale * l;
    if (nl < e->lower) rc_enc_carry(e);
    e->lower = nl;
    e->range = scale * (uint64_t)(r - l);
    if (e->range < ((uint64_t)1 << 32)) {
        rc_enc_push(e, (uint32_t)(e->lower >> 32));
        e->lower <<= 32;
        e->range <<= 32;
    }
    e->nsym++;
}
static void rc_enc_seal(RcEnc *e) {
    if (!e->nsym) return;
    uint64_t point = e->lower + (((uint64_t)1 << 32) - 1);
    if (point < e->lower) rc_enc_carry(e);
    rc_enc_push(e, (uint32_t)(point >> 32));
}

/* ------------------------------------------------------------------------------------ */
static inline uint64_t splitmix64(uint64_t *s) {
    uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

int64_t cco_latent_layout(const CcoDesc *d, int64_t offsets[CCO_MAX_GRIDS]) {
    int64_t p = 0;
    for (int g = d->n_grids - 1; g >= 0; g--) {
        if (offsets) offsets[g] = p;
        p += (int64_t)d->grid_h[g] * d->grid_w[g];
    }
    return p;
}

/* Entropy (de)coding of all grids: component/coolchic.py:72-166 + latent.py:18-187.
 * mode 0 decode (rd), 1 encode given latents (en), 2 sample from the model then encode. */
typedef struct {
    int mode;
    RcDec *rd;
    RcEnc *en;
    uint64_t prng;
    int64_t max_acc, max_hid, n_diag;
} Coder;

static int code_all_grids(const CcoDesc *d, const int64_t *nn, Coder *cd, int8_t *lat) {
    NNLayout L;
    int rc = nn_layout(d, &L);
    if (rc) return rc;
    int dim = L.dim;
    if (dim < 1 || dim > 71) return CCO_ERR_ARG;
    /* the IFCE context plane of grid g has grid g+1's size and is read at (y >> 1, x >> 1): a grid less than half
     * the next finer one (a gap between the latent and hyperlatent resolutions) cannot be read */
    for (int g = 0; d->flag_ifce && g + 1 < d->n_grids; g++)
        if (2 * d->grid_h[g + 1] < d->grid_h[g] || 2 * d->grid_w[g + 1] < d->grid_w[g]) return CCO_ERR_ARG;
    ArmFP arm;
    ArmFP ifce[CCO_MAX_GRIDS];
    memset(ifce, 0, sizeof(ifce));
    {
        const int64_t *qw[8], *qb[8];
        for (int l = 0; l < L.n_arm_lin; l++) {
            qw[l] = nn + L.off_arm_w[l];
            qb[l] = nn + L.off_arm_b[l];
        }
        const int64_t *qws = d->arm_stab ? nn + L.off_arm_w[L.n_arm_lin] : NULL;
        const int64_t *qbs = d->arm_stab ? nn + L.off_arm_b[L.n_arm_lin] : NULL;
        /* component/coolchic.py:72-77 */
        rc = armfp_build(&arm, dim, d->arm_hidden, 2, qw, qb, qws, qbs, d->qshift[0], d->qshift[1],
                         1, d->n_ifce_out, 0);
        if (rc) return rc;
    }
    for (int j = 0; j < L.n_ifce; j++) {
        const int64_t *qw[1] = {nn + L.off_ifce_w[j]};
        const int64_t *qb[1] = {nn + L.off_ifce_b[j]};
        /* component/coolchic.py:114-123 */
        rc = armfp_build(&ifce[j], d->grid_ifce_in[L.ifce_grid[j]], 0, d->n_ifce_out, qw, qb, NULL,
                         NULL, d->qshift[2], d->qshift[3], 0, 0, 1);
        if (rc) return rc;
    }
    int64_t offs[CCO_MAX_GRIDS];
    cco_latent_layout(d, offs);
    int Cf = d->flag_ifce ? d->n_ifce_out : 0;

    for (int g = d->n_grids - 1; g >= 0 && rc == CCO_OK; g--) {
        int h = d->grid_h[g], w = d->grid_w[g];
        int8_t *out = lat + offs[g];
        /* ---- IFCE context plane at the previous grid's resolution (coolchic.py:95-146) */
        int hp, wp;
        int64_t *feat = NULL; /* [hp*wp][Cf] */
        if (Cf > 0) {
            int n_dec = d->n_grids - 1 - g;
            if (n_dec == 0) {
                hp = h;
                wp = w;
            } else {
                hp = d->grid_h[g + 1];
                wp = d->grid_w[g + 1];
            }
            feat = (int64_t *)calloc((size_t)hp * wp * Cf + 1, 8);
            if (!feat) {
                rc = CCO_ERR_NOMEM;
                break;
            }
            int n_in = d->grid_ifce_in[g];
            if (n_in > 0) {
                int j = -1;
                for (int t = 0; t < L.n_ifce; t++)
                    if (L.ifce_grid[t] == g) j = t;
                /* shift of channel c (grid g+1+c) w.r.t. grid g+1: number of size changes
                 * (upsampling.py:575-593, nearest x2 + crop only when shapes differ) */
                int sh[CCO_MAX_GRIDS];
                int n_ch = n_dec > 0 ? n_dec : 1;
                if (n_ch != n_in) {
                    free(feat);
                    rc = CCO_ERR_ARG;
                    break;
                }
                sh[0] = 0;
                for (int c = 1; c < n_ch; c++) {
                    int ga = g + c, gb = g + 1 + c; /* gb coarser-or-equal than ga */
                    int differ = (d->grid_h[ga] != d->grid_h[gb]) || (d->grid_w[ga] != d->grid_w[gb]);
                    sh[c] = sh[c - 1] + (differ ? 1 : 0);
                }
                for (int yy = 0; yy < hp; yy++) {
                    for (int xx = 0; xx < wp; xx++) {
                        int64_t ctx[CCO_MAX_GRIDS], o[32];
                        for (int c = 0; c < n_ch; c++) {
                            if (n_dec == 0) {
                                ctx[c] = 0;
                            } else {
                                int gc = g + 1 + c;
                                ctx[c] = lat[offs[gc] + (int64_t)(yy >> sh[c]) * d->grid_w[gc] + (xx >> sh[c])];
                            }
                        }
                        armfp_forward(&ifce[j], ctx, o, 24, NULL, NULL);
                        for (int f = 0; f < Cf; f++) {
                            /* F.interpolate(x.to(torch.float)).to(int64): fp32 round trip */
                            float fl = (float)o[f];
                            feat[((size_t)yy * wp + xx) * Cf + f] = (int64_t)fl;
                        }
                    }
                }
            }
        }
        /* ---- wavefront over the grid (latent.py:63-173) */
        int Wp = w + 2 * ARM_PAD;
        int32_t *pad = (int32_t *)calloc((size_t)(h + 2 * ARM_PAD) * Wp + 1, 4);
        if (!pad) {
            free(feat);
            rc = CCO_ERR_NOMEM;
            break;
        }
        int64_t n_diag = (w <= ARM_MASK) ? (int64_t)h * w : (int64_t)w + (int64_t)WAVE_STRIDE * (h - 1);
        cd->n_diag += n_diag;
        for (int64_t k = 0; k < n_diag && rc == CCO_OK; k++) {
            int y0, x0, step;
            if (w <= ARM_MASK) { /* raster fallback, latent.py:113-122 */
                y0 = (int)(k / w);
                x0 = (int)(k % w);
                step = 0;
            } else if (k < w) {
                y0 = 0;
                x0 = (int)k;
                step = 1;
            } else {
                y0 = (int)((k - w) / WAVE_STRIDE) + 1;
                x0 = w - WAVE_STRIDE + (int)((k - w) % WAVE_STRIDE);
                step = 1;
            }
            for (int i = 0;; i++) {
                int y = y0 + i, x = x0 - WAVE_STRIDE * i;
                if (i > 0 && (!step || y >= h || x < 0)) break;
                int64_t ctx[80], o[2];
                const int32_t *c = pad + (size_t)(y + ARM_PAD) * Wp + (x + ARM_PAD);
                for (int t = 0; t < d->n_ctx; t++) ctx[t] = c[k_ctx_dy[t] * Wp + k_ctx_dx[t]];
                for (int f = 0; f < Cf; f++)
                    ctx[d->n_ctx + f] = feat[((size_t)(y >> 1) * wp + (x >> 1)) * Cf + f];
                armfp_forward(&arm, ctx, o, 24, &cd->max_acc, &cd->max_hid);
                /* latent.py:165 + rangecoder.py:89-91 (take, mode="clip") */
                int64_t im = o[0] + 16384, is = o[1] + 1280;
                if (im < 0) im = 0;
                if (im > 32767) im = 32767;
                if (is < 0) is = 0;
                if (is > 2560) is = 2560;
                double mu = (double)(float)((double)(im - 16384) / 256.0);
                double b = (double)scale_from_index((int)is);
                int s;
                if (cd->mode == 0) {
                    rc = rc_decode(cd->rd, mu, b, &s);
                    if (rc) break;
                } else {
                    if (cd->mode == 1) {
                        s = out[(size_t)y * w + x];
                    } else {
                        uint32_t q = (uint32_t)(splitmix64(&cd->prng) >> 40), l, r;
                        s = laplace_find(q, mu, b, &l, &r);
                    }
                    rc_encode(cd->en, s, mu, b);
                }
                out[(size_t)y * w + x] = (int8_t)s;
                pad[(size_t)(y + ARM_PAD) * Wp + (x + ARM_PAD)] = s;
            }
        }
        free(pad);
        free(feat);
    }
    armfp_free(&arm);
    for (int j = 0; j < L.n_ifce; j++) armfp_free(&ifce[j]);
    return rc;
}

int cco_decode_latents(const CcoDesc *d, const int64_t *nn, const uint8_t *latent_bytes,
                       size_t nbytes, int8_t *latents_out, int64_t *stats) {
    /* rangecoder.py:80-82: np.frombuffer(raw, uint32) little-endian words */
    size_t nw = nbytes / 4;
    uint32_t *words = (uint32_t *)malloc(nw * 4 + 4);
    if (!words) return CCO_ERR_NOMEM;
    memcpy(words, latent_bytes, nw * 4);
    RcDec rd;
    rc_dec_init(&rd, words, nw);
    Coder cd;
    memset(&cd, 0, sizeof(cd));
    cd.mode = 0;
    cd.rd = &rd;
    int rc = code_all_grids(d, nn, &cd, latents_out);
    if (stats) {
        stats[0] = (int64_t)rd.pos;
        stats[1] = cd.max_acc;
        stats[2] = cd.max_hid;
        stats[3] = cd.n_diag;
    }
    free(words);
    return rc;
}

static int64_t finish_encode(RcEnc *en, uint8_t *out, size_t cap) {
    rc_enc_seal(en);
    int64_t nb = (int64_t)en->n * 4;
    if (en->oom) nb = CCO_ERR_NOMEM;
    else if ((size_t)nb > cap) nb = CCO_ERR_ARG;
    else memcpy(out, en->w, (size_t)nb);
    free(en->w);
    return nb;
}

int64_t cco_encode_latents(const CcoDesc *d, const int64_t *nn, const int8_t *latents, uint8_t *out,
                           size_t cap) {
    int64_t n = cco_latent_layout(d, NULL);
    /* the model has no interval outside [-64, 63]: left(s) = left(s + 1) there, so R would drop to 0 */
    for (int64_t i = 0; i < n; i++)
        if (latents[i] < SYM_MIN || latents[i] > SYM_MAX) return CCO_ERR_ARG;
    int8_t *tmp = (int8_t *)malloc((size_t)n + 1);
    if (!tmp) return CCO_ERR_NOMEM;
    memcpy(tmp, latents, (size_t)n);
    RcEnc en;
    rc_enc_init(&en);
    Coder cd;
    memset(&cd, 0, sizeof(cd));
    cd.mode = 1;
    cd.en = &en;
    int rc = code_all_grids(d, nn, &cd, tmp);
    free(tmp);
    if (rc) {
        free(en.w);
        return rc;
    }
    return finish_encode(&en, out, cap);
}

int64_t cco_sample_latents(const CcoDesc *d, const int64_t *nn, uint64_t seed, int8_t *latents_out,
                           uint8_t *out, size_t cap) {
    RcEnc en;
    rc_enc_init(&en);
    Coder cd;
    memset(&cd, 0, sizeof(cd));
    cd.mode = 2;
    cd.en = &en;
    cd.prng = seed;
    int rc = code_all_grids(d, nn, &cd, latents_out);
    if (rc) {
        free(en.w);
        return rc;
    }
    return finish_encode(&en, out, cap);
}

/* ------------------------------------------------------------------------------------ */
/* Float tail (fp32).  Upsampling in TRAIN-mode kron form (SURVEY F5):
 *   transposed conv  upsampling.py:306-325 ; pre-concat conv upsampling.py:189-196 ;
 *   Upsampling.forward upsampling.py:463-500 ; Synthesis synthesis.py:61-76,272-294.       */
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* y[2m]   = sum_t w[7-2t] x[m-2+t],  y[2m+1] = sum_t w[6-2t] x[m-1+t]  (t=0..3, k=8 case);
 * general even k: P0=k/2, C=2*P0-1+k/2.  2-D kernel K[a][b] = fl(w[a]*w[b]) (torch.kron).
 * in [h][w] -> out [ht][wt] (already cropped to the target size, ht<=2h, wt<=2w).         */
static void convt_kron(const float *in, int h, int w, const float *w1d, int k, float *out, int ht,
                       int wt) {
    int P0 = k / 2, C = 2 * P0 - 1 + k / 2;
#pragma omp parallel for schedule(static)
    for (int u = 0; u < ht; u++) {
        int o1 = u + C;
        int i1_lo = (o1 - (k - 1) + 1) / 2; /* ceil((o1-k+1)/2), o1-k+1 >= 0 here */
        if (o1 - (k - 1) < 0) i1_lo = 0;
        int i1_hi = o1 / 2;
        for (int v = 0; v < wt; v++) {
            int o2 = v + C;
            int i2_lo = (o2 - (k - 1) + 1) / 2;
            if (o2 - (k - 1) < 0) i2_lo = 0;
            int i2_hi = o2 / 2;
            float acc = 0.0f;
            for (int i1 = i1_lo; i1 <= i1_hi; i1++) {
                int a = o1 - 2 * i1;
                int r = clampi(i1 - P0, 0, h - 1);
                for (int i2 = i2_lo; i2 <= i2_hi; i2++) {
                    int b = o2 - 2 * i2;
                    int c = clampi(i2 - P0, 0, w - 1);
                    float kk = w1d[a] * w1d[b];
                    acc = fmaf(kk, in[(size_t)r * w + c], acc);
                }
            }
            out[(size_t)u * wt + v] = acc;
        }
    }
}

/* hi = conv2d(x, kron(w,w), zero padding k/2) + x  (upsampling.py:189-196) */
static void preconcat_kron(const float *in, int h, int w, const float *w1d, int k, float *out) {
    int p = k / 2;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float acc = 0.0f;
            for (int a = 0; a < k; a++) {
                int yy = y + a - p;
                if (yy < 0 || yy >= h) continue;
                for (int b = 0; b < k; b++) {
                    int xx = x + b - p;
                    if (xx < 0 || xx >= w) continue;
                    float kk = w1d[a] * w1d[b];
                    acc = fmaf(kk, in[(size_t)yy * w + xx], acc);
                }
            }
            out[(size_t)y * w + x] = acc + in[(size_t)y * w + x];
        }
}

static void expand_sym(const float *par, int k, float *full) {
    /* _Parameterization_Symmetric_1d.forward, upsampling.py:42-64 */
    int np_ = (k + 1) / 2;
    for (int i = 0; i < np_; i++) full[i] = par[i];
    for (int i = 0; i < k - np_; i++) full[np_ + i] = par[np_ - 1 - (k % 2) - i];
}

/* SynthesisConv2d.forward synthesis.py:61-76: replicate pad, conv + bias, (+x), then ReLU */
static void syn_conv(const float *in, int cin, int h, int w, const float *wt, const float *bias,
                     int cout, int k, int residual, int relu, float *out) {
    int p = (k - 1) / 2;
#pragma omp parallel for collapse(2) schedule(static)
    for (int co = 0; co < cout; co++)
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                float acc = bias[co];
                for (int ci = 0; ci < cin; ci++)
                    for (int ky = 0; ky < k; ky++) {
                        int yy = clampi(y + ky - p, 0, h - 1);
                        for (int kx = 0; kx < k; kx++) {
                            int xx = clampi(x + kx - p, 0, w - 1);
                            acc = fmaf(wt[(((size_t)co * cin + ci) * k + ky) * k + kx],
                                       in[((size_t)ci * h + yy) * w + xx], acc);
                        }
                    }
                if (residual) acc = acc + in[((size_t)co * h + y) * w + x];
                if (relu) acc = acc > 0.0f ? acc : 0.0f;
                out[((size_t)co * h + y) * w + x] = acc;
            }
}

/* ---- F.interpolate(mode = "bilinear" | "bicubic", align_corners=False, antialias=False) ------------
 * Restated from PyTorch's CPU kernel (aten/native/cpu/UpSampleKernel.cpp, generic separable path):
 *   src = fma(scale, dst + 0.5, -0.5) in fp32 (bilinear: max(src, 0)); i0 = min(floor(src), in-1);
 *   lambda = clamp(src - i0, 0, 1); taps clamped to the grid; A = -0.75 cubic coefficients;
 *   value = sum_i wy[i] * (sum_j wx[j] * v[i][j]), products accumulated by an fma chain.
 * scale = 1/scale_factor when a scale factor was given (fixed_upsampling, upsampling.py:586: 0.5),
 * else (float)in / out (component/coolchic.py:187-189).  mode: 1 bilinear, 2 bicubic. */
static float cubic_near(float x);
static float cubic_far(float x);
typedef struct { int idx[4]; float w[4]; } Tap;
static void resize_taps(int in, int out, float scale, int mode, Tap *t) {
    for (int i = 0; i < out; i++) {
        float src = fmaf(scale, (float)i + 0.5f, -0.5f); /* contracted in PyTorch's build */
        if (mode == 1 && src < 0.0f) src = 0.0f;
        int i0 = (int)floorf(src);
        if (i0 > in - 1) i0 = in - 1;
        float lam = src - (float)i0;
        lam = lam < 0.0f ? 0.0f : (lam > 1.0f ? 1.0f : lam);
        if (mode == 1) {
            t[i].idx[0] = i0;
            t[i].idx[1] = i0 + (i0 < in - 1 ? 1 : 0);
            t[i].w[0] = 1.0f - lam;
            t[i].w[1] = lam;
        } else {
            for (int j = 0; j < 4; j++) t[i].idx[j] = clampi(i0 + j - 1, 0, in - 1);
            t[i].w[0] = cubic_far(lam + 1.0f);
            t[i].w[1] = cubic_near(lam);
            float x2 = 1.0f - lam;
            t[i].w[2] = cubic_near(x2);
            t[i].w[3] = cubic_far(x2 + 1.0f);
        }
    }
}
static int resize_torch(const float *in, int c, int h, int w, float *out, int H, int W, int ldH, int ldW, int mode,
                        float sy, float sx) {
    /* writes the top-left H x W (crop) of the resized planes into out[c][ldH][ldW] */
    Tap *ty = (Tap *)malloc(sizeof(Tap) * (size_t)(H + W));
    if (!ty) return CCO_ERR_NOMEM;
    Tap *tx = ty + H;
    resize_taps(h, H, sy, mode, ty);
    resize_taps(w, W, sx, mode, tx);
    const int n = mode == 1 ? 2 : 4;
#pragma omp parallel for collapse(2) schedule(static)
    for (int ch = 0; ch < c; ch++)
        for (int y = 0; y < H; y++) {
            const float *p = in + (size_t)ch * h * w;
            for (int x = 0; x < W; x++) {
                float acc = 0.0f;
                for (int i = 0; i < n; i++) {
                    const float *row = p + (size_t)ty[y].idx[i] * w;
                    float r = tx[x].w[0] * row[tx[x].idx[0]];
                    for (int j = 1; j < n; j++) r = fmaf(tx[x].w[j], row[tx[x].idx[j]], r);
                    acc = (i == 0) ? ty[y].w[0] * r : fmaf(ty[y].w[i], r, acc);
                }
                out[((size_t)ch * ldH + y) * ldW + x] = acc;
            }
        }
    free(ty);
    return CCO_OK;
}
int cco_resize(const float *in, int c, int h, int w, float *out, int H, int W, int mode, int scale_factor_2) {
    if (mode != 1 && mode != 2) return CCO_ERR_ARG;
    float sy = scale_factor_2 ? 0.5f : (float)h / (float)H, sx = scale_factor_2 ? 0.5f : (float)w / (float)W;
    return resize_torch(in, c, h, w, out, H, W, H, W, mode, sy, sx);
}

/* ---- common randomness (--tune=wasserstein): component/core/noise.py:18-55 ------------------------
 * Park-Miller LCG (a = 7^5, m = 2^31 - 1, seed 18101995), two draws per sample, Box-Muller in
 * double precision with pi = 3.14159265359 (log / cos = the canonical ones of detmath.h), rounded to fp32.
 * The fp32 samples equal those of the libm calls the reference makes (math.log / math.cos / math.sqrt)
 * except where the float64 value lies within a few float64 ulp of an fp32 rounding tie: none of the
 * first 12 000 000 samples, one sample (k = 302 383 943) over the whole period (tests/test_detmath.py).
 * One grid per latent resolution (core/coolchic.py:187-191: ceil(img / 2^i)), finest first;
 * fixed_upsampling(bicubic) (upsampling.py:556-595) and a final bicubic interpolate to the image size
 * (bitstream/component/coolchic.py:180-183).  out: [n][H][W], n = latent_res_hi - latent_res_lo + 1. */

/* Samples [first, first + n) of the generator: sample k draws seeds 2k + 1 and 2k + 2 of the sequence */
int cco_noise_samples(uint64_t first, size_t n, float *out) {
    const uint64_t a = 16807ULL, m = 2147483647ULL;
    const double pi = 3.14159265359;
    if (!out || n > (1ULL << 62) || first > (1ULL << 62) - n) return CCO_ERR_ARG;
    uint64_t seed = 18101995ULL, b = a;  /* seed_{2 first} = a^(2 first) seed_0 mod m */
    for (uint64_t e = 2 * first; e; e >>= 1) {
        if (e & 1) seed = (seed * b) % m;
        b = (b * b) % m;
    }
    for (size_t k = 0; k < n; k++) {
        seed = (a * seed) % m;
        double u1 = (double)seed / (double)m;
        seed = (a * seed) % m;
        double u2 = (double)seed / (double)m;
        out[k] = (float)(sqrt(-2 * ccdm_log(u1)) * ccdm_cos(2 * pi * u2));
    }
    return CCO_OK;
}

int cco_cr_noise(const CcoDesc *d, float *out) {
    const int n = d->latent_res_hi - d->latent_res_lo + 1;
    if (n < 1 || n > CCO_MAX_GRIDS) return CCO_ERR_ARG;
    const int H = d->img_h, W = d->img_w;
    int gh[CCO_MAX_GRIDS], gw[CCO_MAX_GRIDS];
    float *g[CCO_MAX_GRIDS];
    uint64_t first = 0;
    for (int i = 0; i < n; i++) g[i] = NULL;
    int rc = CCO_OK;
    for (int i = 0; i < n && rc == CCO_OK; i++) {
        const int sh = d->latent_res_lo + i;
        gh[i] = (int)ceil((double)H / (double)(1LL << sh));
        gw[i] = (int)ceil((double)W / (double)(1LL << sh));
        size_t cnt = (size_t)gh[i] * gw[i];
        g[i] = (float *)malloc(cnt * 4 + 16);
        if (!g[i]) { rc = CCO_ERR_NOMEM; break; }
        rc = cco_noise_samples(first, cnt, g[i]);
        first += cnt;
    }
    /* cascade, coarsest first; cur holds cc planes of size ch x cw */
    float *cur = NULL, *nxt = NULL;
    int ch = 0, cw = 0, cc = 0;
    if (rc == CCO_OK) {
        size_t plane0 = (size_t)gh[0] * gw[0];
        cur = (float *)malloc(plane0 * (size_t)n * 4 + 16);
        nxt = (float *)malloc(plane0 * (size_t)n * 4 + 16);
        if (!cur || !nxt) rc = CCO_ERR_NOMEM;
    }
    if (rc == CCO_OK) {
        ch = gh[n - 1]; cw = gw[n - 1]; cc = 1;
        memcpy(cur, g[n - 1], (size_t)ch * cw * 4);
        for (int i = n - 2; i >= 0 && rc == CCO_OK; i--) {
            const int th = gh[i], tw = gw[i];
            memcpy(nxt, g[i], (size_t)th * tw * 4);
            if (th != ch || tw != cw) {
                /* interpolate(scale_factor=2) gives 2ch x 2cw >= th x tw, cropped */
                if (th > 2 * ch || tw > 2 * cw) { rc = CCO_ERR_ARG; break; }
                rc = resize_torch(cur, cc, ch, cw, nxt + (size_t)th * tw, th, tw, th, tw, 2, 0.5f, 0.5f);
            } else {
                memcpy(nxt + (size_t)th * tw, cur, (size_t)cc * ch * cw * 4);
            }
            float *t = cur; cur = nxt; nxt = t;
            ch = th; cw = tw; cc++;
        }
    }
    if (rc == CCO_OK) {
        if (ch == H && cw == W) memcpy(out, cur, (size_t)n * H * W * 4); /* bicubic at scale 1 = identity */
        else rc = resize_torch(cur, n, ch, cw, out, H, W, H, W, 2, (float)ch / (float)H, (float)cw / (float)W);
    }
    for (int i = 0; i < n; i++) free(g[i]);
    free(cur); free(nxt);
    return rc;
}

int cco_synthesize(const CcoDesc *d, const int64_t *nn, const int8_t *latents, float *out,
                   float *dense_opt) {
    NNLayout L;
    int rc = nn_layout(d, &L);
    if (rc) return rc;
    if (d->ups_k < 4 || (d->ups_k & 1) || !(d->ups_pre_k & 1) || d->ups_k > 15 || d->ups_pre_k > 15)
        return CCO_ERR_ARG;
    int64_t offs[CCO_MAX_GRIDS];
    cco_latent_layout(d, offs);
    /* non-hyper grids, finest first (component/coolchic.py:175) */
    int gl[CCO_MAX_GRIDS], nl = 0;
    for (int g = 0; g < d->n_grids; g++)
        if (!d->grid_is_hyper[g]) gl[nl++] = g;
    const int cr = d->common_randomness != 0;
    if (nl * (cr ? 2 : 1) != d->syn_in) return CCO_ERR_ARG;
    float qs_uw = ldexpf(1.0f, d->qshift[4]);
    float qs_sw = ldexpf(1.0f, d->qshift[6]), qs_sb = ldexpf(1.0f, d->qshift[7]);
    int h0 = d->grid_h[gl[0]], w0 = d->grid_w[gl[0]];
    size_t plane0 = (size_t)h0 * w0;
    if (cr && (h0 != d->img_h || w0 != d->img_w || nl != d->latent_res_hi - d->latent_res_lo + 1))
        return CCO_ERR_ARG; /* the reference concatenates noise at image size with the dense latent */
    float *cur = (float *)malloc(plane0 * (size_t)(2 * nl + 1) * 4 + 16);
    float *nxt = (float *)malloc(plane0 * (size_t)(2 * nl + 1) * 4 + 16);
    if (!cur || !nxt) {
        free(cur);
        free(nxt);
        return CCO_ERR_NOMEM;
    }
    /* start from the coarsest */
    int gc = gl[nl - 1];
    int ch = d->grid_h[gc], cw = d->grid_w[gc], cc = 1;
    for (size_t i = 0; i < (size_t)ch * cw; i++) cur[i] = (float)latents[offs[gc] + i];
    for (int idx = 0; idx < nl - 1; idx++) {
        int gt = gl[nl - 2 - idx];
        int th = d->grid_h[gt], tw = d->grid_w[gt];
        float wt_par[8], wc_par[8], wt_full[16], wc_full[16];
        int kid = idx % d->n_ups;
        for (int i = 0; i < L.kt_par; i++) wt_par[i] = (float)nn[L.off_ups_tw + (int64_t)kid * L.kt_par + i] * qs_uw;
        for (int i = 0; i < L.kc_par; i++) wc_par[i] = (float)nn[L.off_ups_cw + (int64_t)kid * L.kc_par + i] * qs_uw;
        expand_sym(wt_par, d->ups_k, wt_full);
        expand_sym(wc_par, d->ups_pre_k, wc_full);
        /* channel 0: high branch of the target grid */
        float *tgt = (float *)malloc((size_t)th * tw * 4 + 16);
        if (!tgt) {
            free(cur);
            free(nxt);
            return CCO_ERR_NOMEM;
        }
        for (size_t i = 0; i < (size_t)th * tw; i++) tgt[i] = (float)latents[offs[gt] + i];
        preconcat_kron(tgt, th, tw, wc_full, d->ups_pre_k, nxt);
        free(tgt);
        for (int c = 0; c < cc; c++)
            convt_kron(cur + (size_t)c * ch * cw, ch, cw, wt_full, d->ups_k, nxt + (size_t)(c + 1) * th * tw, th, tw);
        float *t = cur;
        cur = nxt;
        nxt = t;
        ch = th;
        cw = tw;
        cc++;
    }
    if (cr) {
        /* bitstream/component/coolchic.py:179-183: noise channels appended to the dense latent */
        rc = cco_cr_noise(d, cur + plane0 * (size_t)nl);
        if (rc) {
            free(cur);
            free(nxt);
            return rc;
        }
    }
    if (dense_opt) memcpy(dense_opt, cur, plane0 * (size_t)d->syn_in * 4);
    /* ---- synthesis */
    int C = L.syn_c_out;
    int maxc = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++)
        if (d->syn_out[l] > maxc) maxc = d->syn_out[l];
    float *a = (float *)malloc(plane0 * (size_t)maxc * 4 + 16);
    float *b = (float *)malloc(plane0 * (size_t)maxc * 4 + 16);
    float *stab = (float *)malloc(plane0 * (size_t)C * 4 + 16);
    float *wbuf = (float *)malloc(((size_t)128 * 128 * 15 * 15 + 128) * 4);
    if (!a || !b || !stab || !wbuf) {
        free(a); free(b); free(stab); free(wbuf); free(cur); free(nxt);
        return CCO_ERR_NOMEM;
    }
    float bbuf[128];
    if (d->syn_stab) {
        size_t nw = (size_t)C * L.syn_stab_in;
        for (size_t i = 0; i < nw; i++) wbuf[i] = (float)nn[L.off_syn_st_w + (int64_t)i] * qs_sw;
        for (int i = 0; i < C; i++) bbuf[i] = (float)nn[L.off_syn_st_b + i] * qs_sb;
        syn_conv(cur, L.syn_stab_in, h0, w0, wbuf, bbuf, C, 1, 0, 0, stab);
    }
    memcpy(a, cur, plane0 * (size_t)d->syn_in * 4);
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        int k = d->syn_k[l], co = d->syn_out[l];
        size_t nw = (size_t)co * in_ft * k * k;
        for (size_t i = 0; i < nw; i++) wbuf[i] = (float)nn[L.off_syn_w[l] + (int64_t)i] * qs_sw;
        for (int i = 0; i < co; i++) bbuf[i] = (float)nn[L.off_syn_b[l] + i] * qs_sb;
        if (d->syn_res[l] && co != in_ft) {
            free(a); free(b); free(stab); free(wbuf); free(cur); free(nxt);
            return CCO_ERR_ARG;
        }
        syn_conv(a, in_ft, h0, w0, wbuf, bbuf, co, k, d->syn_res[l], d->syn_relu[l], b);
        float *t = a;
        a = b;
        b = t;
        in_ft = co;
    }
    if (d->syn_stab)
        for (size_t i = 0; i < plane0 * (size_t)C; i++) a[i] = a[i] + stab[i];
    /* output_transform, synthesis.py:294 */
    for (size_t i = 0; i < (size_t)C * C; i++) wbuf[i] = (float)nn[L.off_syn_ot_w + (int64_t)i] * qs_sw;
    for (int i = 0; i < C; i++) bbuf[i] = (float)nn[L.off_syn_ot_b + i] * qs_sb;
    syn_conv(a, C, h0, w0, wbuf, bbuf, C, 1, 0, 0, b);
    /* final interpolate + crop, component/coolchic.py:187-192 */
    int H = d->img_h, W = d->img_w;
    rc = CCO_OK;
    if (h0 == H && w0 == W) {
        /* every mode is the identity at scale 1 (bicubic weights are exactly 0,1,0,0) */
        memcpy(out, b, plane0 * (size_t)C * 4);
    } else if (d->final_ups == 0) {
        /* legacy "nearest": src = min(floor(dst * (in/out as fp32)), in-1) */
        float sy = (float)h0 / (float)H, sx = (float)w0 / (float)W;
        for (int c = 0; c < C; c++)
            for (int y = 0; y < H; y++) {
                int yy = (int)floorf((float)y * sy);
                if (yy > h0 - 1) yy = h0 - 1;
                for (int x = 0; x < W; x++) {
                    int xx = (int)floorf((float)x * sx);
                    if (xx > w0 - 1) xx = w0 - 1;
                    out[((size_t)c * H + y) * W + x] = b[((size_t)c * h0 + yy) * w0 + xx];
                }
            }
    } else {
        /* size is given -> scale = in / out; output is exactly img size, nothing to crop */
        rc = resize_torch(b, C, h0, w0, out, H, W, H, W, d->final_ups == 1 ? 1 : 2, (float)h0 / (float)H,
                          (float)w0 / (float)W);
    }
    free(a); free(b); free(stab); free(wbuf); free(cur); free(nxt);
    return rc;
}

/* bitstream/decode.py:191-206 (+ io/format/yuv.py:274-300 avg_pool2d 2x2, :239-256 clamp) */
int cco_finish_frame(const float *in, int h, int w, int bitdepth, int data_type, float *out_a,
                     float *out_b, float *out_c) {
    float M = (float)((1 << bitdepth) - 1);
    size_t n = (size_t)h * w;
    if (data_type != 1) {
        for (size_t i = 0; i < 3 * n; i++) {
            float v = rintf(M * in[i]) / M;
            v = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
            out_a[i] = rintf(v * M) / M;
        }
        return CCO_OK;
    }
    for (size_t i = 0; i < n; i++) {
        float v = rintf(M * in[i]) / M;
        v = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
        out_a[i] = rintf(v * M) / M;
    }
    int h2 = h / 2, w2 = w / 2;
    for (int c = 1; c < 3; c++) {
        float *o = (c == 1) ? out_b : out_c;
        const float *p = in + (size_t)c * n;
        for (int y = 0; y < h2; y++)
            for (int x = 0; x < w2; x++) {
                float s = 0.0f;
                for (int dy = 0; dy < 2; dy++)
                    for (int dx = 0; dx < 2; dx++)
                        s += rintf(M * p[(size_t)(2 * y + dy) * w + 2 * x + dx]) / M;
                float v = s / 4.0f;
                v = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
                o[(size_t)y * w2 + x] = rintf(v * M) / M;
            }
    }
    return CCO_OK;
}

/* ---- P/B prediction --------------------------------------------------------------------
 * bitstream/decode.py:156-189.  apply_global_translation (globalmotion.py:151-160) is a
 * grid_sample(nearest, border, align_corners=True) by an integer flow: an integer shift with
 * border clamp.  Warper.forward (warp.py:294-397) runs in its TRAINING branch at decode time
 * (SURVEY F5): no 1/64-pel flow quantisation; filter_size >= 6 -> windowed sinc (warp.py:226-268):
 * integer part by clamped gathers, fractional part by N taps cos(pi(s-k)/N) * sinc(s-k),
 * first along x (flow channel 0) for each of the N rows, then along y (flow channel 1).
 * Coefficients are evaluated in double precision with the canonical sin / cos of detmath.h (exactly
 * reproducible on the GPU) and rounded to fp32; the reference does it in fp32 with its platform's libm.
 * The two are at most 3 fp32 ulp apart for N = 6 ... 14, more than 1 ulp at 12 % (N = 6) to 32 % (N = 14) of
 * the offsets (tests/test_detmath.py); products and sums are fp32, sequential, unfused.            */
static void sinc_coeffs(float s, int n, float *c) {
    const float PIf = 3.14159265358979323846f;
    int lt = -(n / 2) + 1;
    for (int k = 0; k < n; k++) {
        float arg = s - (float)(lt + k);
        float pa = PIf * arg;
        double win = ccdm_cos((double)(pa / (float)n));
        double sc = (arg == 0.0f) ? 1.0 : ccdm_sin((double)pa) / (double)pa;
        c[k] = (float)win * (float)sc;
    }
}

/* Debug images of the canonical functions, for comparison with the device (tests/test_detmath.py):
 * y[i] = sin / cos / log (fn 0 / 1 / 2) of x[i]; c[N i + k] = tap k of the N-tap windowed sinc at offset s[i]. */
int cco_detmath(int fn, const double *x, double *y, size_t n) {
    if (fn < 0 || fn > 2 || !x || !y) return CCO_ERR_ARG;
    for (size_t i = 0; i < n; i++) y[i] = fn == 0 ? ccdm_sin(x[i]) : (fn == 1 ? ccdm_cos(x[i]) : ccdm_log(x[i]));
    return CCO_OK;
}
int cco_sinc_coeffs(int taps, const float *s, float *c, size_t n) {
    if (taps < 6 || taps > 14 || (taps & 1) || !s || !c) return CCO_ERR_ARG;
    for (size_t i = 0; i < n; i++) sinc_coeffs(s[i], taps, c + (size_t)taps * i);
    return CCO_OK;
}

static void warp_sinc(const float *ref, int h, int w, int gx, int gy, const float *flow, int n, float *out) {
    /* ref [3][h][w]; flow [2][h][w] (0: horizontal, 1: vertical); out [3][h][w] */
    size_t plane = (size_t)h * w;
    int lt = -(n / 2) + 1;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float fx = flow[(size_t)y * w + x], fy = flow[plane + (size_t)y * w + x];
            float rx = floorf(fx), ry = floorf(fy);
            float cx[16], cy[16];
            sinc_coeffs(fx - rx, n, cx);
            sinc_coeffs(fy - ry, n, cy);
            int xs[16], ys[16];
            for (int k = 0; k < n; k++) {
                /* neighbour index clamped to the frame (warp.py:352-358), then the global
                 * shift of the reference, clamped as well (globalmotion.py:154-155) */
                float nx = (float)x + (float)(lt + k) + rx, ny = (float)y + (float)(lt + k) + ry;
                nx = nx < 0.0f ? 0.0f : (nx > (float)(w - 1) ? (float)(w - 1) : nx);
                ny = ny < 0.0f ? 0.0f : (ny > (float)(h - 1) ? (float)(h - 1) : ny);
                xs[k] = clampi((int)nx + gx, 0, w - 1);
                ys[k] = clampi((int)ny + gy, 0, h - 1);
            }
            for (int c = 0; c < 3; c++) {
                const float *p = ref + (size_t)c * plane;
                float col = 0.0f;
                for (int i = 0; i < n; i++) {
                    float line = 0.0f;
                    for (int j = 0; j < n; j++) {
                        float t = p[(size_t)ys[i] * w + xs[j]] * cx[j];
                        line = (j == 0) ? t : line + t;
                    }
                    float t2 = line * cy[i];
                    col = (i == 0) ? t2 : col + t2;
                }
                out[(size_t)c * plane + (size_t)y * w + x] = col;
            }
        }
}

/* filter_size 2 / 4: WarpParameter picks "torch_bilinear" / "torch_bicubic" (warp.py:50-56), i.e.
 * F.grid_sample(padding_mode="border", align_corners=True) on backward_grid + flow / ((size-1)/2)
 * (warp.py:92-111, 314-334).  Restated from PyTorch's CPU kernels:
 *  - torch.linspace(-1, 1, n) (RangeFactoriesKernel.cpp): step = 2/(n-1) in fp32;
 *    i < n/2 ? fma(step, i, -1) : fma(-step, n-1-i, 1)   (checked == torch for n = 2..400, 768..4096)
 *  - unnormalise: (g + 1) * ((size-1)/2); border: clip to [0, size-1] (GridSamplerKernel.cpp)
 *  - bilinear: weights s*e, s*w, n*e, n*w; value = fma chain nw -> ne -> sw -> se (bit-exact with
 *    torch 2.11 on random inputs, oracle/gen_golden_gop.py)
 *  - bicubic: A = -0.75 cubic convolution coefficients of t = x - floor(x) (unclipped), each of the
 *    4x4 taps clipped to the frame; within 2e-7 of torch (its exact contraction pattern is
 *    compiler dependent). */
static float lin_coord(int n, int i) {
    float step = 2.0f / (float)(n - 1);
    return (i < n / 2) ? fmaf(step, (float)i, -1.0f) : fmaf(-step, (float)(n - 1 - i), 1.0f);
}
static float cubic_near(float x) { /* |x| <= 1: ((A+2)x - (A+3)) x x + 1 */
    float a = 1.25f * x - 2.25f;
    float b = a * x;
    return fmaf(b, x, 1.0f);
}
static float cubic_far(float x) { /* 1 < |x| < 2: ((Ax - 5A) x + 8A) x - 4A */
    float a = -0.75f * x + 3.75f;
    float b = a * x + -6.0f;
    return b * x + 3.0f;
}
static void warp_grid(const float *ref, int h, int w, int gx, int gy, const float *flow, int n, float *out) {
    size_t plane = (size_t)h * w;
    const float sx = (float)((w - 1.0) / 2.0), sy = (float)((h - 1.0) / 2.0);
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float fx = flow[(size_t)y * w + x], fy = flow[plane + (size_t)y * w + x];
            float g0 = lin_coord(w, x) + fx / sx, g1 = lin_coord(h, y) + fy / sy;
            float ix = (g0 + 1.0f) * sx, iy = (g1 + 1.0f) * sy;
            if (n == 2) {
                ix = fminf((float)(w - 1), fmaxf(ix, 0.0f));
                iy = fminf((float)(h - 1), fmaxf(iy, 0.0f));
                float xw = floorf(ix), yn = floorf(iy);
                float ww = ix - xw, e = 1.0f - ww, nn = iy - yn, s = 1.0f - nn;
                float k_nw = s * e, k_ne = s * ww, k_sw = nn * e, k_se = nn * ww;
                int x0 = (int)xw, y0 = (int)yn, x1 = x0 + 1, y1 = y0 + 1;
                int xa = clampi(x0 + gx, 0, w - 1), xb = clampi((x1 < w ? x1 : w - 1) + gx, 0, w - 1);
                int ya = clampi(y0 + gy, 0, h - 1), yb = clampi((y1 < h ? y1 : h - 1) + gy, 0, h - 1);
                for (int c = 0; c < 3; c++) {
                    const float *p = ref + (size_t)c * plane;
                    float v00 = p[(size_t)ya * w + xa];
                    float v01 = x1 < w ? p[(size_t)ya * w + xb] : 0.0f;
                    float v10 = y1 < h ? p[(size_t)yb * w + xa] : 0.0f;
                    float v11 = (x1 < w && y1 < h) ? p[(size_t)yb * w + xb] : 0.0f;
                    float r = v00 * k_nw;
                    r = fmaf(v01, k_ne, r);
                    r = fmaf(v10, k_sw, r);
                    r = fmaf(v11, k_se, r);
                    out[(size_t)c * plane + (size_t)y * w + x] = r;
                }
            } else {
                float fxx = floorf(ix), fyy = floorf(iy);
                float tx = ix - fxx, ty = iy - fyy;
                float cx[4] = {cubic_far(tx + 1.0f), cubic_near(tx), cubic_near(1.0f - tx), cubic_far(2.0f - tx)};
                float cy[4] = {cubic_far(ty + 1.0f), cubic_near(ty), cubic_near(1.0f - ty), cubic_far(2.0f - ty)};
                int xs[4], ys[4];
                for (int k = 0; k < 4; k++) {
                    float nx = fminf((float)(w - 1), fmaxf(fxx + (float)(k - 1), 0.0f));
                    float ny = fminf((float)(h - 1), fmaxf(fyy + (float)(k - 1), 0.0f));
                    xs[k] = clampi((int)nx + gx, 0, w - 1);
                    ys[k] = clampi((int)ny + gy, 0, h - 1);
                }
                for (int c = 0; c < 3; c++) {
                    const float *p = ref + (size_t)c * plane;
                    float rows[4];
                    for (int i = 0; i < 4; i++) {
                        const float *q = p + (size_t)ys[i] * w;
                        float r = cx[0] * q[xs[0]];
                        r = fmaf(cx[1], q[xs[1]], r);
                        r = fmaf(cx[2], q[xs[2]], r);
                        r = fmaf(cx[3], q[xs[3]], r);
                        rows[i] = r;
                    }
                    float a = cy[0] * rows[0];
                    a = fmaf(cy[1], rows[1], a);
                    a = fmaf(cy[2], rows[2], a);
                    a = fmaf(cy[3], rows[3], a);
                    out[(size_t)c * plane + (size_t)y * w + x] = a;
                }
            }
        }
}

int cco_inter_predict(const float *residue, const float *motion, const float *ref0,
                      const float *ref1, int h, int w, int is_b, const int32_t *global_flow,
                      int warp_filter_size, float *out) {
    if (warp_filter_size < 2 || (warp_filter_size & 1) || warp_filter_size > 16) return CCO_ERR_UNSUPPORTED;
    if (warp_filter_size < 6 && (h < 2 || w < 2)) return CCO_ERR_UNSUPPORTED;
    size_t plane = (size_t)h * w;
    float *w0 = (float *)malloc(plane * 3 * 4 + 16), *w1 = NULL;
    if (!w0) return CCO_ERR_NOMEM;
    void (*warp)(const float *, int, int, int, int, const float *, int, float *) =
        warp_filter_size < 6 ? warp_grid : warp_sinc;
    warp(ref0, h, w, global_flow[0], global_flow[1], motion, warp_filter_size, w0);
    if (is_b) {
        w1 = (float *)malloc(plane * 3 * 4 + 16);
        if (!w1) {
            free(w0);
            return CCO_ERR_NOMEM;
        }
        warp(ref1, h, w, global_flow[2], global_flow[3], motion + 2 * plane, warp_filter_size, w1);
    }
    for (size_t i = 0; i < plane; i++) {
        float a = residue[3 * plane + i] + 0.5f;
        a = a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a);
        float b = 0.0f;
        if (is_b) {
            b = residue[4 * plane + i] + 0.5f;
            b = b < 0.0f ? 0.0f : (b > 1.0f ? 1.0f : b);
        }
        for (int c = 0; c < 3; c++) {
            float pred = w0[c * plane + i];
            if (is_b) {
                float t1 = b * pred, t2 = (1.0f - b) * w1[c * plane + i];
                pred = t1 + t2;
            }
            float m = a * pred;
            out[c * plane + i] = m + residue[c * plane + i];
        }
    }
    free(w0);
    free(w1);
    return CCO_OK;
}
