// ccd_api.cu -- host side of libccdec.so: the C-ABI of include/ccdec.h.
//
// Host work per Cool-chic (all tiny, <= a few kB): exp-Golomb decode of the NN payload
// (neuralnet.py:92-204, expgolomb.py:74-130), conversion of the ARM / IFCE integers into
// fixed-point parameters (armint.py:30-170) packed for the entropy kernel, a worst-case
// bound analysis that proves the int32-operand fast path safe (otherwise the generic int64
// kernel is used -- still on the GPU), dequantisation of upsampling / synthesis weights.
// Everything per-pixel runs in ccd_entropy.cu / ccd_synth.cu.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "ccd_internal.h"

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return fail(CCD_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                        __FILE__, __LINE__);                                                   \
    } while (0)

const uint32_t k_scale_bits[CCD_N_SCALE] = {
#include "ccd_scale_table.inc"
};

// ---- NN integer layout (neuralnet.py:120-148; module order arm, ifce, upsampling, synthesis;
// per module all weights then all biases; parameter registration order of each module) --------
struct NNLayout {
    int dim = 0, n_arm_lin = 0;
    int64_t arm_w[9] = {0}, arm_b[9] = {0};  // [n_arm_lin] = stabiliser
    int n_ifce = 0;
    int ifce_grid[CCD_MAX_GRIDS] = {0};
    int64_t ifce_w[CCD_MAX_GRIDS] = {0}, ifce_b[CCD_MAX_GRIDS] = {0};
    int kt_par = 0, kc_par = 0;
    int64_t ups_tw = 0, ups_cw = 0;
    int syn_c = 0, syn_stab_in = 0;
    int64_t syn_ot_w = 0, syn_st_w = 0, syn_w[CCD_MAX_SYN] = {0};
    int64_t syn_ot_b = 0, syn_st_b = 0, syn_b[CCD_MAX_SYN] = {0};
    int64_t counts[8] = {0};
    int64_t total = 0;
};

int validate_desc(const CcdCoolChicDesc *d) {
    if (!d) return fail(CCD_ERR_ARG, "null descriptor");
    if (d->n_grids < 1 || d->n_grids > CCD_MAX_GRIDS) return fail(CCD_ERR_ARG, "n_grids=%d out of range", d->n_grids);
    if (d->n_syn_layers < 1 || d->n_syn_layers > CCD_MAX_SYN)
        return fail(CCD_ERR_ARG, "n_syn_layers=%d out of range", d->n_syn_layers);
    if (d->arm_hidden < 0 || d->arm_hidden > 7) return fail(CCD_ERR_ARG, "arm_hidden=%d out of range", d->arm_hidden);
    if (d->n_ctx < 0 || d->n_ctx > 40) return fail(CCD_ERR_ARG, "n_ctx=%d out of range", d->n_ctx);
    if (d->n_ifce_out < 0 || d->n_ifce_out > 31) return fail(CCD_ERR_ARG, "n_ifce_out=%d out of range", d->n_ifce_out);
    if (d->n_ctx + d->n_ifce_out < 1) return fail(CCD_ERR_ARG, "ARM without any context");
    if (d->img_h < 1 || d->img_w < 1) return fail(CCD_ERR_ARG, "bad image size");
    for (int g = 0; g < d->n_grids; g++) {
        if (d->grid_h[g] < 1 || d->grid_w[g] < 1) return fail(CCD_ERR_ARG, "grid %d has an empty dimension", g);
        if (d->grid_ifce_in[g] < 0 || d->grid_ifce_in[g] > 31) return fail(CCD_ERR_ARG, "grid %d: bad ifce_in", g);
        if (d->flag_ifce && d->grid_ifce_in[g] > 0 && d->grid_ifce_in[g] != std::max(d->n_grids - 1 - g, 1))
            return fail(CCD_ERR_ARG, "grid %d: ifce_in=%d inconsistent", g, d->grid_ifce_in[g]);
    }
    for (int i = 0; i < 8; i++) {
        if (d->expgol[i] < 0 || d->expgol[i] > 12) return fail(CCD_ERR_ARG, "exp-Golomb order out of range");
        if (d->qshift[i] > 0 || d->qshift[i] < -24) return fail(CCD_ERR_ARG, "q_step out of range");
    }
    if (d->qshift[0] < -8 || d->qshift[2] < -8 || d->qshift[1] < -16 || d->qshift[3] < -16)
        return fail(CCD_ERR_ARG, "ARM/IFCE q_step out of range");
    if (d->ups_k < 4 || (d->ups_k & 1) || d->ups_k > 14) return fail(CCD_ERR_ARG, "ups_k=%d unsupported", d->ups_k);
    if (!(d->ups_pre_k & 1) || d->ups_pre_k > 15 || d->ups_pre_k < 1)
        return fail(CCD_ERR_ARG, "ups_pre_k=%d unsupported", d->ups_pre_k);
    for (int l = 0; l < d->n_syn_layers; l++) {
        if (d->syn_out[l] < 1 || d->syn_out[l] > 127 || d->syn_k[l] < 1 || !(d->syn_k[l] & 1))
            return fail(CCD_ERR_ARG, "synthesis layer %d malformed", l);
    }
    return CCD_OK;
}

int nn_layout(const CcdCoolChicDesc *d, NNLayout *L) {
    int rc = validate_desc(d);
    if (rc) return rc;
    int64_t p = 0, q;
    const int dim = d->n_ctx + d->n_ifce_out;
    L->dim = dim;
    L->n_arm_lin = d->arm_hidden + 1;
    for (int l = 0; l < L->n_arm_lin; l++) {
        L->arm_w[l] = p;
        p += (int64_t)((l == d->arm_hidden) ? 2 : dim) * dim;
    }
    if (d->arm_stab) {
        L->arm_w[L->n_arm_lin] = p;
        p += 2 * dim;
    }
    L->counts[0] = p;
    q = p;
    for (int l = 0; l < L->n_arm_lin; l++) {
        L->arm_b[l] = p;
        p += (l == d->arm_hidden) ? 2 : dim;
    }
    if (d->arm_stab) {
        L->arm_b[L->n_arm_lin] = p;
        p += 2;
    }
    L->counts[1] = p - q;
    q = p;
    if (d->flag_ifce)
        for (int g = 0; g < d->n_grids; g++)
            if (d->grid_ifce_in[g] > 0) {
                L->ifce_grid[L->n_ifce] = g;
                L->ifce_w[L->n_ifce++] = p;
                p += (int64_t)d->n_ifce_out * d->grid_ifce_in[g];
            }
    L->counts[2] = p - q;
    q = p;
    for (int j = 0; j < L->n_ifce; j++) {
        L->ifce_b[j] = p;
        p += d->n_ifce_out;
    }
    L->counts[3] = p - q;
    L->kt_par = (d->ups_k + 1) / 2;
    L->kc_par = (d->ups_pre_k + 1) / 2;
    q = p;
    L->ups_tw = p;
    p += (int64_t)d->n_ups * L->kt_par;
    L->ups_cw = p;
    p += (int64_t)d->n_ups * L->kc_par;
    L->counts[4] = p - q;
    L->counts[5] = 2 * (int64_t)d->n_ups;  // one (unused) bias per kernel, upsampling.py:123,243
    p += L->counts[5];
    const int C = d->syn_out[d->n_syn_layers - 1];
    L->syn_c = C;
    L->syn_stab_in = d->common_randomness ? d->syn_in / 2 : d->syn_in;
    q = p;
    L->syn_ot_w = p;
    p += (int64_t)C * C;
    if (d->syn_stab) {
        L->syn_st_w = p;
        p += (int64_t)C * L->syn_stab_in;
    }
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        L->syn_w[l] = p;
        p += (int64_t)d->syn_out[l] * in_ft * d->syn_k[l] * d->syn_k[l];
        in_ft = d->syn_out[l];
    }
    L->counts[6] = p - q;
    q = p;
    L->syn_ot_b = p;
    p += C;
    if (d->syn_stab) {
        L->syn_st_b = p;
        p += C;
    }
    for (int l = 0; l < d->n_syn_layers; l++) {
        L->syn_b[l] = p;
        p += d->syn_out[l];
    }
    L->counts[7] = p - q;
    L->total = p;
    return CCD_OK;
}

// MSB-first exp-Golomb reader over the NN payload
int64_t decode_nn_host(const CcdCoolChicDesc *d, const NNLayout &L, const uint8_t *bytes, size_t nbytes,
                       int64_t *out) {
    const size_t nbits = nbytes * 8;
    size_t pos = (size_t)d->nn_n_bit_pad;
    auto bit = [&](size_t i) -> int { return (bytes[i >> 3] >> (7 - (i & 7))) & 1; };
    int64_t n = 0;
    for (int m = 0; m < 8; m++) {
        const int k = d->expgol[m];
        for (int64_t i = 0; i < L.counts[m]; i++) {
            int z = 0;
            while (pos < nbits && bit(pos) == 0) {
                z++;
                pos++;
            }
            if (pos + (size_t)z + 1 + (size_t)k > nbits || z > 60)
                return fail(CCD_ERR_NN_TRUNCATED, "NN payload truncated at parameter %lld", (long long)n);
            uint64_t val = 0;
            for (int j = 0; j <= z; j++) val = (val << 1) | (uint64_t)bit(pos++);
            uint64_t rem = 0;
            for (int j = 0; j < k; j++) rem = (rem << 1) | (uint64_t)bit(pos++);
            const int64_t v = (int64_t)(((val - 1) << k) + rem);
            out[n++] = (v & 1) ? (v + 1) / 2 : -(v / 2);
        }
    }
    return n;
}

// ---- fixed-point ARM parameters (armint.py:30-170) ------------------------------------------
struct ArmInts {
    int dim = 0, n_hidden = 0, n_out = 2;
    std::vector<std::vector<int64_t>> W;  // per linear layer, TRANSPOSED: [in][out]
    std::vector<std::vector<int64_t>> B;
    std::vector<int64_t> Ws, Bs;          // stabiliser [in][n_out], [n_out] (zeros if absent)
};

ArmInts build_arm(int dim, int n_hidden, int n_out, const int64_t *const *qw, const int64_t *const *qb,
                  const int64_t *qws, const int64_t *qbs, int s_w, int s_b, bool subtract_last,
                  int n_inter_ft, bool no_residual) {
    ArmInts a;
    a.dim = dim;
    a.n_hidden = n_hidden;
    a.n_out = n_out;
    a.W.resize(n_hidden + 1);
    a.B.resize(n_hidden + 1);
    for (int l = 0; l <= n_hidden; l++) {
        const int out = (l == n_hidden) ? n_out : dim;
        a.W[l].assign((size_t)dim * out, 0);
        a.B[l].assign((size_t)out, 0);
        for (int o = 0; o < out; o++) {
            for (int i = 0; i < dim; i++) {
                const bool ifce_col = n_inter_ft > 0 && l == 0 && i >= dim - n_inter_ft;
                const int shift = 16 + s_w - (ifce_col ? 8 : 0);
                int64_t v = qw[l][(size_t)o * dim + i] * ((int64_t)1 << shift);
                // every square layer is residual: +I folded into the weights (armint.py:114-124)
                if (out == dim && !no_residual && o == i) v += (int64_t)1 << (ifce_col ? 8 : 16);
                a.W[l][(size_t)i * out + o] = v;
            }
            int64_t qv = qb[l][o];
            if (l == n_hidden && subtract_last && o == 1) qv -= (int64_t)4 << (-s_b);  // armint.py:98-100
            a.B[l][o] = qv * ((int64_t)1 << (32 + s_b));
        }
    }
    a.Ws.assign((size_t)dim * n_out, 0);
    a.Bs.assign((size_t)n_out, 0);
    if (qws) {
        for (int o = 0; o < n_out; o++) {
            for (int i = 0; i < dim; i++) {
                const bool ifce_col = n_inter_ft > 0 && i >= dim - n_inter_ft;
                a.Ws[(size_t)i * n_out + o] = qws[(size_t)o * dim + i] * ((int64_t)1 << (16 + s_w - (ifce_col ? 8 : 0)));
            }
            a.Bs[o] = qbs[o] * ((int64_t)1 << (32 + s_b));
        }
    }
    return a;
}

typedef __int128 i128;
inline i128 iabs128(int64_t v) { return v < 0 ? -(i128)v : (i128)v; }

// worst-case |IFCE feature| (8 fractional bits), incl. the fp32 round trip
bool ifce_bound(const ArmInts &a, i128 *bound) {
    i128 best = 0;
    for (int o = 0; o < a.n_out; o++) {
        i128 acc = iabs128(a.B[0][o]);
        for (int i = 0; i < a.dim; i++) {
            if (iabs128(a.W[0][(size_t)i * a.n_out + o]) > INT32_MAX) return false;
            acc += iabs128(a.W[0][(size_t)i * a.n_out + o]) * ((i128)64 << 16);
        }
        if (acc >= ((i128)1 << 62)) return false;
        i128 f = (acc >> 24) + 1;
        f += (f >> 22) + 1;  // float rounding
        best = std::max(best, f);
    }
    *bound = best;
    return true;
}

// Can the ARM run with int32 operands (weights, activations) and int64 accumulators?
bool arm_fits_int32(const ArmInts &a, int n_ctx, i128 ifce_feat_bound) {
    std::vector<i128> X((size_t)a.dim);
    for (int i = 0; i < a.dim; i++) X[i] = (i < n_ctx) ? ((i128)64 << 16) : (ifce_feat_bound << 16);
    for (int i = 0; i < a.dim; i++)
        if (X[i] > INT32_MAX) return false;
    auto layer_ok = [&](const std::vector<int64_t> &W, const std::vector<int64_t> &B, int out,
                        const std::vector<i128> &Xin, std::vector<i128> *acc) {
        acc->assign((size_t)out, 0);
        for (int o = 0; o < out; o++) {
            i128 s = iabs128(B[o]);
            for (int i = 0; i < a.dim; i++) {
                if (iabs128(W[(size_t)i * out + o]) > INT32_MAX) return false;
                s += iabs128(W[(size_t)i * out + o]) * Xin[i];
            }
            if (s >= ((i128)1 << 61)) return false;
            (*acc)[o] = s;
        }
        return true;
    };
    std::vector<i128> acc, stab;
    if (!layer_ok(a.Ws, a.Bs, a.n_out, X, &stab)) return false;
    for (int l = 0; l < a.n_hidden; l++) {
        if (!layer_ok(a.W[l], a.B[l], a.dim, X, &acc)) return false;
        for (int o = 0; o < a.dim; o++) {
            X[o] = acc[o] >> 16;
            if (X[o] > INT32_MAX) return false;
        }
    }
    if (!layer_ok(a.W[a.n_hidden], a.B[a.n_hidden], a.n_out, X, &acc)) return false;
    return true;
}

void put_i32(std::vector<unsigned char> &b, int64_t v) {
    int32_t t = (int32_t)v;
    b.insert(b.end(), (unsigned char *)&t, (unsigned char *)&t + 4);
}
void put_i64(std::vector<unsigned char> &b, int64_t v) { b.insert(b.end(), (unsigned char *)&v, (unsigned char *)&v + 8); }
void pad_to(std::vector<unsigned char> &b, size_t a) {
    while (b.size() % a) b.push_back(0);
}

void pack_arm(const ArmInts &a, bool fast, std::vector<unsigned char> &b) {
    const int dim = a.dim;
    if (fast) {
        const int opm = (dim + 3) / 4, opmp = opm <= 2 ? 2 : (opm <= 4 ? 4 : 8), dimp = 4 * opm;
        for (int l = 0; l < a.n_hidden; l++)
            for (int i = 0; i < dim; i++)
                for (int m = 0; m < 4; m++)
                    for (int o = 0; o < opmp; o++) {
                        const int out = m * opm + o;
                        put_i32(b, (o < opm && out < dim) ? a.W[l][(size_t)i * dim + out] : 0);
                    }
        for (int i = 0; i < dimp; i++)
            for (int o = 0; o < 2; o++) put_i32(b, i < dim ? a.W[a.n_hidden][(size_t)i * 2 + o] : 0);
        for (int i = 0; i < dimp; i++)
            for (int o = 0; o < 2; o++) put_i32(b, i < dim ? a.Ws[(size_t)i * 2 + o] : 0);
        pad_to(b, 8);
        for (int l = 0; l < a.n_hidden; l++)
            for (int o = 0; o < dimp; o++) put_i64(b, o < dim ? a.B[l][o] : 0);
    } else {
        for (int l = 0; l < a.n_hidden; l++)
            for (size_t t = 0; t < (size_t)dim * dim; t++) put_i64(b, a.W[l][t]);
        for (size_t t = 0; t < (size_t)dim * 2; t++) put_i64(b, a.W[a.n_hidden][t]);
        for (size_t t = 0; t < (size_t)dim * 2; t++) put_i64(b, a.Ws[t]);
        for (int l = 0; l < a.n_hidden; l++)
            for (int o = 0; o < dim; o++) put_i64(b, a.B[l][o]);
    }
    put_i64(b, a.B[a.n_hidden][0]);
    put_i64(b, a.B[a.n_hidden][1]);
    put_i64(b, a.Bs[0]);
    put_i64(b, a.Bs[1]);
    pad_to(b, 16);
}

void pack_ifce(const ArmInts &a, bool fast, std::vector<unsigned char> &b) {
    const int n_in = a.dim, cf = a.n_out, cfp = (cf + 3) & ~3;
    if (fast) {
        for (int i = 0; i < n_in; i++)
            for (int o = 0; o < cfp; o++) put_i32(b, o < cf ? a.W[0][(size_t)i * cf + o] : 0);
        pad_to(b, 8);
    } else {
        for (size_t t = 0; t < (size_t)n_in * cf; t++) put_i64(b, a.W[0][t]);
    }
    for (int o = 0; o < cf; o++) put_i64(b, a.B[0][o]);
    pad_to(b, 16);
}

int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

struct DeviceBuf {
    unsigned char *p = nullptr;
    size_t cap = 0;
};

struct PreparedJob {
    CcdJob *job = nullptr;
    const CcdCoolChicDesc *d = nullptr;
    NNLayout L;
    std::vector<int64_t> nn;
    std::vector<unsigned char> blob;
    EntStream es;
    bool fast = false;
    size_t smem = 0;
    int64_t n_sym = 0;
    int64_t lat_off_by_grid[CCD_MAX_GRIDS];
    bool pad_lat = false;   // latents owned by the library: every grid starts on a 16-byte boundary (TMA source)
    int64_t lat_bytes = 0;  // bytes of the latent buffer in that layout
    int nl = 0, gl[CCD_MAX_GRIDS];  // latent grids (not hyper), finest first
    bool resized = false;   // the finest latent grid is smaller than the image: the output is computed at its size
    const int8_t *lat[CCD_MAX_GRIDS];  // the device latents the float tail reads for each grid
    // float tail (plan_tail)
    bool tail = false;      // goes through the batched path
    int tail_cinp = 0, tail_C = 0;
    size_t off_tailP = 0, off_tailQ = 0, off_tailRaw = 0;  // inside the batched path's scratch
    // device offsets inside the upload arena
    size_t off_words = 0, off_blob = 0, off_syn = 0, off_lat = 0;
    std::vector<float> syn_f;  // dequantised synthesis weights, packed
    size_t syn_off_ot_w = 0, syn_off_ot_b = 0, syn_off_st_w = 0, syn_off_st_b = 0;
    size_t syn_off_w[CCD_MAX_SYN], syn_off_b[CCD_MAX_SYN];
};

}  // namespace

struct CcdContext {
    int device = 0;
    float *d_scale = nullptr;
    uint32_t *d_cdf = nullptr;
    DeviceBuf upload;   // words / blobs / stream structs / statuses / synthesis weights
    DeviceBuf scratch;  // synthesis intermediates, latents when the caller does not want them, MS-SSIM pyramid levels
    DeviceBuf zeros;    // all zero: the latents of the grids a synthesis job masks
    unsigned char *h_pin = nullptr;
    size_t h_pin_cap = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    float last_ms[4] = {0, 0, 0, 0};
    int32_t last_status[16] = {0};
    uint64_t last_upload_bytes = 0;
    uint32_t prod_mask = 0x3777u;  // warps 3, 7, 11 stay idle: the coder warp (15) owns its scheduler
    int n_sm = 132;
    // entropy launches of different ARM architectures (e.g. intra / residue / motion streams of a GOP) run
    // side by side on these streams: each launch only fills as many SMs as it has streams
    cudaStream_t aux[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_join[3] = {nullptr, nullptr, nullptr};
};

namespace {

// Entry points run on the context's device and put the caller's current device back on return (the host
// application -- PyTorch -- keeps its own notion of the current device).
struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = (prev == dev) || cudaSetDevice(dev) == cudaSuccess;
        if (prev == dev) prev = -1;  // nothing to restore
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

int ensure_dev(DeviceBuf &b, size_t bytes) {
    if (bytes <= b.cap) return CCD_OK;
    if (b.p) CUDA_TRY(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = bytes + bytes / 4 + (1 << 20);
    CUDA_TRY(cudaMalloc(&b.p, want));
    b.cap = want;
    return CCD_OK;
}

inline size_t al(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// The staging of one job call: inputs, then one results region, at the same offsets in the pinned buffer (h) and the
// upload arena (dv).  One copy takes the inputs and the initial result values up, one brings the results back.
struct Arena {
    size_t end = 0;
    unsigned char *h = nullptr, *dv = nullptr;
    size_t take(size_t bytes, size_t align = 256) {
        const size_t at = al(end, align);
        end = at + bytes;
        return at;
    }
};

// Reserves the pinned staging buffer and the upload arena for everything A has laid out
int stage(CcdContext *c, Arena &A) {
    if (A.end > c->h_pin_cap) {
        if (c->h_pin) CUDA_TRY(cudaFreeHost(c->h_pin));
        c->h_pin = nullptr;
        c->h_pin_cap = 0;
        const size_t want = A.end + A.end / 4 + (1 << 16);
        CUDA_TRY(cudaMallocHost(&c->h_pin, want));
        c->h_pin_cap = want;
    }
    if (int rc = ensure_dev(c->upload, A.end)) return rc;
    A.h = c->h_pin;
    A.dv = c->upload.p;
    return CCD_OK;
}

// Copies the results region [off, A.end) back to the pinned buffer and waits for the call to finish
int download(const Arena &A, size_t off, cudaStream_t st, const char *what) {
    CUDA_TRY(cudaMemcpyAsync(A.h + off, A.dv + off, A.end - off, cudaMemcpyDeviceToHost, st));
    const cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return fail(CCD_ERR_CUDA, "%s execution failed: %s", what, cudaGetErrorString(se));
    return CCD_OK;
}

// A job's status from its result words: a decode job's is word [0] of its entropy status words.  A job with a bad_index
// gets the smallest bad index the kernel found, ~0 (bad_index -1) when there is none; any other one is CCD_ERR_ARG.
int job_status(CcdJob &, const int32_t (&words)[16]) { return words[0]; }
int job_status(CcdSynthJob &, const int32_t &word) { return word; }
template <class Job> int job_status(Job &J, const unsigned long long &bad) {
    J.bad_index = (int64_t)bad;
    return bad == ~0ull ? CCD_OK : CCD_ERR_ARG;
}

// The per-job results of a job call from its downloaded result words (result[i]: job i's).  Sets each failing job's
// status; returns CCD_OK, or the first failing job's status with the message say(i) gives it through fail().
template <class Job, class Word, class Say>
int report(Job *jobs, int n_jobs, const Word *result, Say &&say) {
    int first = CCD_OK;
    for (int i = 0; i < n_jobs; i++) {
        const int s = job_status(jobs[i], result[i]);
        if (s == CCD_OK) continue;
        jobs[i].status = s;
        if (!first) first = say(i);
    }
    return first;
}

// f64 partials added in order, part[0], part[stride], ..., part[(n - 1) * stride]: the same sum on every run
double ordered_sum(const double *part, size_t n, size_t stride = 1) {
    double s = 0.0;
    for (size_t t = 0; t < n; t++) s += part[t * stride];
    return s;
}

// The body of every entry point that takes a context: body(stream) runs on the context's device, and a failing call
// leaves the context quiescent -- the pinned staging buffer, the upload arena and the scratch may be reused (or
// re-allocated) by the next call -- with its own message kept.
template <class F>
int guarded(CcdContext *ctx, void *cuda_stream, F &&body) {
    if (!ctx) return fail(CCD_ERR_ARG, "null context");
    DeviceGuard guard(ctx->device);
    if (!guard.ok) return fail(CCD_ERR_CUDA, "cudaSetDevice(%d) failed", ctx->device);
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    const int rc = body(st);
    if (rc != CCD_OK) {
        const std::string keep = g_err;
        cudaStreamSynchronize(st);
        for (int a = 0; a < 3; a++)
            if (ctx->aux[a]) cudaStreamSynchronize(ctx->aux[a]);
        cudaGetLastError();
        g_err = keep;
    }
    return rc;
}

// A call on a job array: checks the list, sets every job's status to CCD_OK, runs body(stream) through guarded()
template <class Job, class F>
int job_call(CcdContext *ctx, Job *jobs, int n_jobs, void *cuda_stream, F &&body) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(CCD_ERR_ARG, "bad job list");
        for (int i = 0; i < n_jobs; i++) jobs[i].status = CCD_OK;
        return n_jobs == 0 ? CCD_OK : body(st);
    });
}

// Shared memory of the entropy kernel for one stream (DESIGN §4.1): sets S.ring and S.rows, returns the bytes.  The
// row ring holds every row the wavefront still reads (row y - 4 runs 40 columns ahead of row y), so its size follows
// from the width alone.  The window ring takes 2 slots per symbol of the longest diagonal + 64, up to 1024, and is
// halved, down to 64 slots, while the whole does not fit: the producers wait for free slots, so a smaller ring only
// lets fewer symbols run ahead of the coder.  More than CCD_SMEM_MAX bytes: not even a 64-slot ring fits.
size_t plan_entropy_smem(EntStream &S, int n_max, int rows_need) {
    S.rows = next_pow2(rows_need);
    S.ring = std::min(1024, std::max(64, next_pow2(2 * n_max + 64)));
    size_t smem = ccd_entropy_smem_bytes(S.ring, S.rows, S.arm_blob_bytes, S.ifce_blob_max);
    while (smem > CCD_SMEM_MAX && S.ring > 64) {
        S.ring /= 2;
        smem = ccd_entropy_smem_bytes(S.ring, S.rows, S.arm_blob_bytes, S.ifce_blob_max);
    }
    return smem;
}
int entropy_smem_ok(size_t smem) {
    if (smem <= CCD_SMEM_MAX) return CCD_OK;
    return fail(CCD_ERR_UNSUPPORTED, "the entropy stage needs %zu bytes of shared memory, %d are available", smem,
                CCD_SMEM_MAX);
}

// Host preparation of the float tail of one job: NN integers, latent layout, dequantised synthesis weights.
int prepare_synthesis(PreparedJob &P, const int64_t *nn_ints_opt) {
    const CcdCoolChicDesc *d = P.d;
    int rc = nn_layout(d, &P.L);
    if (rc) return rc;
    const NNLayout &L = P.L;
    P.nn.resize((size_t)L.total);
    if (nn_ints_opt) {
        memcpy(P.nn.data(), nn_ints_opt, (size_t)L.total * 8);
    } else {
        int64_t n = decode_nn_host(d, L, P.job->nn_bytes, P.job->nn_nbytes, P.nn.data());
        if (n < 0) return (int)n;
    }
    const int64_t *nn = P.nn.data();
    // ---- latent layout (decode order: coarsest first)
    int64_t off = 0, nsym = 0;
    for (int g = d->n_grids - 1; g >= 0; g--) {
        if (P.pad_lat) off = (off + 15) & ~(int64_t)15;
        P.lat_off_by_grid[g] = off;
        off += (int64_t)d->grid_h[g] * d->grid_w[g];
        nsym += (int64_t)d->grid_h[g] * d->grid_w[g];
    }
    P.n_sym = nsym;
    P.lat_bytes = off;
    P.nl = 0;
    for (int g = 0; g < d->n_grids; g++)
        if (!d->grid_is_hyper[g]) P.gl[P.nl++] = g;
    P.resized = P.nl > 0 && (d->grid_h[P.gl[0]] != d->img_h || d->grid_w[P.gl[0]] != d->img_w);
    if (off >= ((int64_t)1 << 31)) return fail(CCD_ERR_UNSUPPORTED, "more than 2^31 latent symbols");
    // ---- synthesis weights, dequantised (neuralnet.py:185-190: float32(int) * q_step)
    const float qs_w = ldexpf(1.0f, d->qshift[6]), qs_b = ldexpf(1.0f, d->qshift[7]);
    std::vector<float> &F = P.syn_f;
    F.clear();
    auto push = [&](int64_t off0, int64_t n, float qs) {
        size_t at = F.size();
        for (int64_t i = 0; i < n; i++) F.push_back((float)nn[off0 + i] * qs);
        while (F.size() % 4) F.push_back(0.0f);
        return at;
    };
    const int C = L.syn_c;
    P.syn_off_ot_w = push(L.syn_ot_w, (int64_t)C * C, qs_w);
    P.syn_off_ot_b = push(L.syn_ot_b, C, qs_b);
    if (d->syn_stab) {
        P.syn_off_st_w = push(L.syn_st_w, (int64_t)C * L.syn_stab_in, qs_w);
        P.syn_off_st_b = push(L.syn_st_b, C, qs_b);
    }
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        P.syn_off_w[l] = push(L.syn_w[l], (int64_t)d->syn_out[l] * in_ft * d->syn_k[l] * d->syn_k[l], qs_w);
        P.syn_off_b[l] = push(L.syn_b[l], d->syn_out[l], qs_b);
        if (d->syn_res[l] && d->syn_out[l] != in_ft) return fail(CCD_ERR_ARG, "residual layer %d changes width", l);
        in_ft = d->syn_out[l];
    }
    return CCD_OK;
}

// Host preparation of one job: prepare_synthesis, then the entropy stage's ARM / IFCE packing and stream descriptor.
int prepare_job(PreparedJob &P, const int64_t *nn_ints_opt) {
    if (int rc = prepare_synthesis(P, nn_ints_opt)) return rc;
    const CcdCoolChicDesc *d = P.d;
    const NNLayout &L = P.L;
    const int64_t *nn = P.nn.data();
    // ---- ARM + IFCE integers
    const int dim = L.dim;
    std::vector<const int64_t *> qw, qb;
    for (int l = 0; l < L.n_arm_lin; l++) {
        qw.push_back(nn + L.arm_w[l]);
        qb.push_back(nn + L.arm_b[l]);
    }
    // component/coolchic.py:72-77
    ArmInts arm = build_arm(dim, d->arm_hidden, 2, qw.data(), qb.data(),
                            d->arm_stab ? nn + L.arm_w[L.n_arm_lin] : nullptr,
                            d->arm_stab ? nn + L.arm_b[L.n_arm_lin] : nullptr, d->qshift[0], d->qshift[1], true,
                            d->n_ifce_out, false);
    std::vector<ArmInts> ifce;
    i128 feat_bound = 0;
    bool fast = ccd_entropy_has_fast(d->n_ctx, d->n_ifce_out);
    for (int j = 0; j < L.n_ifce; j++) {
        const int64_t *w1[1] = {nn + L.ifce_w[j]};
        const int64_t *b1[1] = {nn + L.ifce_b[j]};
        // component/coolchic.py:114-123
        ifce.push_back(build_arm(d->grid_ifce_in[L.ifce_grid[j]], 0, d->n_ifce_out, w1, b1, nullptr, nullptr,
                                 d->qshift[2], d->qshift[3], false, 0, true));
        i128 bnd = 0;
        if (!ifce_bound(ifce.back(), &bnd)) fast = false;
        if (d->grid_ifce_in[L.ifce_grid[j]] > CCD_IFCE_FAST_MAX) fast = false;
        feat_bound = std::max(feat_bound, bnd);
    }
    if (fast) fast = arm_fits_int32(arm, d->n_ctx, feat_bound);
    P.fast = fast;
    P.blob.clear();
    pack_arm(arm, fast, P.blob);
    const int arm_bytes = (int)P.blob.size();

    EntStream &S = P.es;
    memset(&S, 0, sizeof(S));
    S.n_grids = d->n_grids;
    S.n_ctx = d->n_ctx;
    S.cf = d->flag_ifce ? d->n_ifce_out : 0;
    if (!d->flag_ifce && d->n_ifce_out != 0) return fail(CCD_ERR_ARG, "n_ifce_out without flag_ifce");
    S.n_hidden = d->arm_hidden;
    S.has_ifce = d->flag_ifce;
    S.arm_blob_bytes = arm_bytes;
    S.n_symbols = P.n_sym;
    int n_max = 1, rows_need = 8, ifce_max = 0;
    for (int gi = 0; gi < d->n_grids; gi++) {
        const int g = d->n_grids - 1 - gi;  // fine-first index
        EntGrid &G = S.grid[gi];
        G.h = d->grid_h[g];
        G.w = d->grid_w[g];
        G.raster = G.w <= 9;
        G.n_diag = G.raster ? G.h * G.w : G.w + CCD_MASK_STRIDE * (G.h - 1);
        G.lat_off = P.lat_off_by_grid[g];
        G.n_dec = gi;
        G.ifce_in = d->flag_ifce ? d->grid_ifce_in[g] : 0;
        G.ifce_blob_off = 0;
        G.ifce_blob_bytes = 0;
        if (G.ifce_in > 0) {
            int j = -1;
            for (int t = 0; t < L.n_ifce; t++)
                if (L.ifce_grid[t] == g) j = t;
            G.ifce_blob_off = (int)P.blob.size();
            pack_ifce(ifce[(size_t)j], fast, P.blob);
            G.ifce_blob_bytes = (int)P.blob.size() - G.ifce_blob_off;
            ifce_max = std::max(ifce_max, G.ifce_blob_bytes);
            // channel c <- grid g+1+c, nearest-upsampled to grid g+1's size
            // (core/upsampling.py:575-593: x2 + crop only when consecutive shapes differ)
            const int n_ch = G.ifce_in;
            int sh = 0;
            for (int c = 0; c < n_ch; c++) {
                if (gi == 0) {  // nothing decoded yet: a single all-zero channel (coolchic.py:95-96)
                    G.ch_sh[c] = -1;
                    G.ch_w[c] = 1;
                    G.ch_off[c] = 0;
                    continue;
                }
                const int gc = g + 1 + c;
                if (c > 0) {
                    const int ga = g + c;
                    if (d->grid_h[ga] != d->grid_h[gc] || d->grid_w[ga] != d->grid_w[gc]) sh++;
                }
                G.ch_sh[c] = sh;
                G.ch_w[c] = d->grid_w[gc];
                G.ch_off[c] = P.lat_off_by_grid[gc];
            }
        }
        const int nk = G.raster ? 1 : std::min(G.h, (G.w + CCD_MASK_STRIDE - 1) / CCD_MASK_STRIDE);
        n_max = std::max(n_max, nk);
        rows_need = std::max(rows_need, G.raster ? 8 : (G.w - 1) / CCD_MASK_STRIDE + 6);
    }
    S.ifce_blob_max = ifce_max;
    P.smem = plan_entropy_smem(S, n_max, rows_need);

    return CCD_OK;
}

// Device scratch of the float tail of one job on the per-stream path.
struct SynScratch {
    size_t off_nxt = 0, off_a = 0, off_b = 0, off_stab = 0, off_noise_raw = 0, off_noise_a = 0, off_noise_b = 0, total = 0;
    std::vector<int> pw2;  // layer l is evaluated together with l + 1 by k_syn_pw2 (two 1x1 layers)
};
SynScratch syn_scratch_plan(const CcdCoolChicDesc *d) {
    SynScratch S;
    int nl = 0, g0 = -1;
    for (int g = 0; g < d->n_grids; g++)
        if (!d->grid_is_hyper[g]) {
            if (g0 < 0) g0 = g;
            nl++;
        }
    S.pw2.assign((size_t)std::max(d->n_syn_layers, 1), 0);
    if (g0 < 0 || d->n_syn_layers < 1) return S;
    const size_t plane = (size_t)d->grid_h[g0] * d->grid_w[g0];
    const int C = d->syn_out[d->n_syn_layers - 1];
    int maxc = std::max(d->syn_in, C);
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        const bool can = l + 1 < d->n_syn_layers && d->syn_k[l] == 1 && d->syn_k[l + 1] == 1 && !d->syn_res[l] &&
                         !d->syn_res[l + 1] && in_ft <= 16 && d->syn_out[l + 1] <= 8;
        if (can) {
            S.pw2[(size_t)l] = 1;
            maxc = std::max(maxc, d->syn_out[l + 1]);
            in_ft = d->syn_out[l + 1];
            l++;
        } else {
            maxc = std::max(maxc, d->syn_out[l]);
            in_ft = d->syn_out[l];
        }
    }
    const size_t dense = al(plane * (size_t)(std::max(nl, d->syn_in) + 1) * 4);
    const size_t trunk = al(plane * (size_t)maxc * 4);
    size_t p = dense;
    S.off_nxt = p; p += dense;
    S.off_a = p; p += trunk;
    S.off_b = p; p += trunk;
    S.off_stab = p; p += al(plane * (size_t)C * 4);
    if (d->common_randomness) {
        S.off_noise_raw = p; p += al(plane * 2 * 4 + (size_t)nl * 64);  // sum of ceil(H/2^i) ceil(W/2^i) <= 2 plane
        S.off_noise_a = p; p += al(plane * (size_t)nl * 4);
        S.off_noise_b = p; p += al(plane * (size_t)nl * 4);
    }
    S.total = p;
    return S;
}

void expand_sym(const float *par, int k, float *full) {
    // _Parameterization_Symmetric_1d (core/upsampling.py:42-64): a b c d -> a b c d [d] c b a
    const int np = (k + 1) / 2;
    for (int i = 0; i < np; i++) full[i] = par[i];
    for (int i = 0; i < k - np; i++) full[np + i] = par[np - 1 - (k % 2) - i];
}

// Full 1-D taps of cascade level idx (level 0 upsamples the coarsest grid): quantised parameters -> dequantised ->
// expand_sym
void level_taps(const PreparedJob &P, int idx, float full_t[16], float full_c[16]) {
    const CcdCoolChicDesc *d = P.d;
    const NNLayout &L = P.L;
    const float qs_uw = ldexpf(1.0f, d->qshift[4]);
    const int kid = idx % d->n_ups;
    float par_t[8], par_c[8];
    for (int i = 0; i < L.kt_par; i++) par_t[i] = (float)P.nn[(size_t)(L.ups_tw + (int64_t)kid * L.kt_par + i)] * qs_uw;
    for (int i = 0; i < L.kc_par; i++) par_c[i] = (float)P.nn[(size_t)(L.ups_cw + (int64_t)kid * L.kc_par + i)] * qs_uw;
    expand_sym(par_t, d->ups_k, full_t);
    expand_sym(par_c, d->ups_pre_k, full_c);
}

// The synthesis of a job as layer descriptors with their weights at d_synw (null when only the shapes are needed)
struct SynNet {
    SynLayerDev layers[CCD_MAX_SYN], stab, ot;
};
SynNet syn_net(const PreparedJob &P, const float *d_synw) {
    const CcdCoolChicDesc *d = P.d;
    const int C = P.L.syn_c;
    auto at = [&](size_t off) { return d_synw ? d_synw + off : nullptr; };
    SynNet N;
    int in_ft = d->syn_in;
    for (int l = 0; l < d->n_syn_layers; l++) {
        N.layers[l] = SynLayerDev{in_ft, d->syn_out[l], d->syn_k[l], d->syn_res[l], d->syn_relu[l], at(P.syn_off_w[l]),
                                  at(P.syn_off_b[l])};
        in_ft = d->syn_out[l];
    }
    N.stab = SynLayerDev{P.L.syn_stab_in, C, 1, 0, 0, at(P.syn_off_st_w), at(P.syn_off_st_b)};
    N.ot = SynLayerDev{C, C, 1, 0, 0, at(P.syn_off_ot_w), at(P.syn_off_ot_b)};
    return N;
}

// final F.interpolate of an output computed at h0 x w0, smaller than the image (component/coolchic.py:187-192)
int resize_output(const CcdCoolChicDesc *d, const float *src, int C, int h0, int w0, float *dst, cudaStream_t st) {
    int rc;
    if (d->final_ups == 0)
        rc = ccd_resize_nearest(src, C, h0, w0, dst, d->img_h, d->img_w, st);
    else
        rc = ccd_resize_torch(src, C, h0, w0, dst, d->img_h, d->img_w, d->final_ups == 1 ? 1 : 2,
                              (float)h0 / (float)d->img_h, (float)w0 / (float)d->img_w, st);
    return rc ? fail(CCD_ERR_CUDA, "resize launch") : CCD_OK;
}

// Upsampling cascade + synthesis + final resize for one job on the per-stream path (all kernels on `st`).
int run_synthesis(const PreparedJob &P, const float *d_synw, float *d_out, unsigned char *scratch, size_t scratch_bytes,
                  cudaStream_t st) {
    const CcdCoolChicDesc *d = P.d;
    const int cr = d->common_randomness != 0;
    const int nl = P.nl;
    const int *gl = P.gl;
    if (nl * (cr ? 2 : 1) != d->syn_in || nl < 1)
        return fail(CCD_ERR_ARG, "synthesis input width %d does not match %d latent grids", d->syn_in, nl);
    const int h0 = d->grid_h[gl[0]], w0 = d->grid_w[gl[0]];
    if (cr && (h0 != d->img_h || w0 != d->img_w || nl != d->latent_res_hi - d->latent_res_lo + 1))
        return fail(CCD_ERR_ARG, "common randomness needs a full-resolution finest latent grid");
    const size_t plane = (size_t)h0 * w0;
    const int C = P.L.syn_c;
    const SynScratch SS = syn_scratch_plan(d);
    if (SS.total > scratch_bytes) return fail(CCD_ERR_NOMEM, "internal: scratch too small (%zu > %zu)", SS.total, scratch_bytes);
    float *cur = reinterpret_cast<float *>(scratch);
    float *nxt = reinterpret_cast<float *>(scratch + SS.off_nxt);
    float *bufa = reinterpret_cast<float *>(scratch + SS.off_a);
    float *bufb = reinterpret_cast<float *>(scratch + SS.off_b);
    float *stab = reinterpret_cast<float *>(scratch + SS.off_stab);

    int gc = gl[nl - 1];
    int ch = d->grid_h[gc], cw = d->grid_w[gc], cc = 1;
    int rc;
    if ((rc = ccd_ups_first(P.lat[gc], ch, cw, cur, st))) return fail(CCD_ERR_CUDA, "ups_first launch");
    for (int idx = 0; idx < nl - 1; idx++) {
        const int gt = gl[nl - 2 - idx];
        const int th = d->grid_h[gt], tw = d->grid_w[gt];
        if (th > 2 * ch || tw > 2 * cw) return fail(CCD_ERR_ARG, "grid %d more than twice the size of its parent", gt);
        float full_t[16], full_c[16];
        level_taps(P, idx, full_t, full_c);
        if (d->ups_k == 8 && d->ups_pre_k == 7) {
            if ((rc = ccd_ups_level(P.lat[gt], th, tw, cur, cc, ch, cw, full_t, full_c, nxt, st)))
                return fail(CCD_ERR_CUDA, "ups_level launch");
        } else {
            if ((rc = ccd_ups_pre(P.lat[gt], th, tw, full_c, d->ups_pre_k, nxt, st)))
                return fail(CCD_ERR_CUDA, "ups_pre launch");
            if ((rc = ccd_ups_convt(cur, cc, ch, cw, full_t, d->ups_k, nxt + (size_t)th * tw, th, tw, st)))
                return fail(CCD_ERR_CUDA, "ups_convt launch");
        }
        std::swap(cur, nxt);
        ch = th;
        cw = tw;
        cc++;
    }
    if (cr) {
        // bitstream/component/coolchic.py:179-183: noise grids (noise.py) -> fixed_upsampling(bicubic)
        // (upsampling.py:556-595) -> channels nl .. 2 nl - 1 of the synthesis input
        float *raw = reinterpret_cast<float *>(scratch + SS.off_noise_raw);
        float *na = reinterpret_cast<float *>(scratch + SS.off_noise_a);
        float *nb = reinterpret_cast<float *>(scratch + SS.off_noise_b);
        int gh[CCD_MAX_GRIDS], gw[CCD_MAX_GRIDS];
        size_t goff[CCD_MAX_GRIDS], tot = 0;
        for (int i = 0; i < nl; i++) {
            const int sh = d->latent_res_lo + i;
            gh[i] = (int)((d->img_h + (1LL << sh) - 1) >> sh);
            gw[i] = (int)((d->img_w + (1LL << sh) - 1) >> sh);
            goff[i] = tot;
            tot += (size_t)gh[i] * gw[i];
        }
        if (ccd_cr_noise(raw, 0, tot, st)) return fail(CCD_ERR_CUDA, "noise launch");
        int nh = gh[nl - 1], nw = gw[nl - 1], nc = 1;
        const float *ncur = raw + goff[nl - 1];
        for (int i = nl - 2; i >= 0; i--) {
            const int th = gh[i], tw = gw[i];
            float *dstp = (i == 0) ? cur + plane * (size_t)nl : ((ncur == na) ? nb : na);
            if (th > 2 * nh || tw > 2 * nw) return fail(CCD_ERR_ARG, "noise grid %d more than twice its parent", i);
            if (cudaMemcpyAsync(dstp, raw + goff[i], (size_t)th * tw * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
                return fail(CCD_ERR_CUDA, "noise copy");
            if (th != nh || tw != nw) {
                if (ccd_resize_torch(ncur, nc, nh, nw, dstp + (size_t)th * tw, th, tw, 2, 0.5f, 0.5f, st))
                    return fail(CCD_ERR_CUDA, "noise upsampling launch");
            } else if (cudaMemcpyAsync(dstp + (size_t)th * tw, ncur, (size_t)nc * nh * nw * 4, cudaMemcpyDeviceToDevice,
                                       st) != cudaSuccess) {
                return fail(CCD_ERR_CUDA, "noise copy");
            }
            ncur = dstp;
            nh = th;
            nw = tw;
            nc++;
        }
        if (nl == 1 &&
            cudaMemcpyAsync(cur + plane, raw, plane * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return fail(CCD_ERR_CUDA, "noise copy");
        // gh[0] x gw[0] == image size here, so the final bicubic interpolate is the identity
    }
    // ---- synthesis (core/synthesis.py:272-294): one kernel in the fused family, else one kernel per layer (two
    // 1x1 layers at a time where k_syn_pw2 takes them)
    const SynNet N = syn_net(P, d_synw);
    const bool same = (h0 == d->img_h && w0 == d->img_w);
    float *ot_dst = same ? d_out : bufa;
    rc = ccd_syn_fused(cur, h0, w0, d->syn_in, N.layers, d->n_syn_layers, d->syn_stab ? &N.stab : nullptr, N.ot, ot_dst, st);
    if (rc > 0) return fail(CCD_ERR_CUDA, "fused synthesis launch");
    if (rc < 0) {
        if (d->syn_stab && (rc = ccd_syn_layer(cur, h0, w0, N.stab, stab, st))) return fail(CCD_ERR_CUDA, "stabiliser launch");
        const float *src = cur;
        float *dst = bufa, *other = bufb;
        for (int l = 0; l < d->n_syn_layers; l++) {
            if (SS.pw2[(size_t)l]) {
                if ((rc = ccd_syn_pointwise2(src, h0, w0, N.layers[l], N.layers[l + 1], dst, st)))
                    return fail(CCD_ERR_CUDA, "pointwise launch");
                l++;
            } else if ((rc = ccd_syn_layer(src, h0, w0, N.layers[l], dst, st))) {
                return fail(CCD_ERR_CUDA, "synthesis layer launch");
            }
            src = dst;
            std::swap(dst, other);
        }
        float *trunk = const_cast<float *>(src);
        if (trunk == cur) return fail(CCD_ERR_ARG, "synthesis without layers");
        if (d->syn_stab)
            if ((rc = ccd_syn_add(trunk, stab, plane * (size_t)C, st))) return fail(CCD_ERR_CUDA, "add launch");
        ot_dst = same ? d_out : dst;
        if ((rc = ccd_syn_layer(trunk, h0, w0, N.ot, ot_dst, st))) return fail(CCD_ERR_CUDA, "output transform launch");
    }
    return same ? CCD_OK : resize_output(d, ot_dst, C, h0, w0, d_out, st);
}

size_t synthesis_scratch_bytes(const CcdCoolChicDesc *d) { return syn_scratch_plan(d).total + 4096; }

// The checks of a job's frame-tail request (job i of its call)
int check_finish(const CcdJob &job, const PreparedJob &J, int i) {
    if (job.finish_bitdepth == 0) return CCD_OK;
    if (job.finish_bitdepth < 1 || job.finish_bitdepth > 16 || job.finish_type < 0 || job.finish_type > 3)
        return fail(CCD_ERR_ARG, "job %d: bad frame tail request (bitdepth %d, type %d)", i, job.finish_bitdepth, job.finish_type);
    if (J.L.syn_c != 3) return fail(CCD_ERR_ARG, "job %d: the frame tail needs a 3-channel output, found %d", i, J.L.syn_c);
    if (job.finish_type == 1 && (!job.d_out_u || !job.d_out_v))
        return fail(CCD_ERR_ARG, "job %d: yuv420 frame tail needs u and v outputs", i);
    return CCD_OK;
}

// decode_frame's frame tail (decode.py:191-206) of a job that asks for it, from its raw output at the image size: the
// finished frame goes to the job's outputs.  (k_tail_syn finishes the full-size outputs it writes itself.)
int finish_job(const CcdJob &job, const float *raw, cudaStream_t st) {
    if (job.finish_bitdepth == 0) return CCD_OK;
    const int ft = job.finish_type == 3 ? 2 : job.finish_type;  // flow: three full planes, as yuv444
    if (ccd_finish(raw, job.desc->img_h, job.desc->img_w, job.finish_bitdepth, ft, job.d_out, job.d_out_u, job.d_out_v, st))
        return fail(CCD_ERR_CUDA, "finish_frame launch failed");
    return CCD_OK;
}

// ---- float tail planning -----------------------------------------------------------------------------------
// A job takes the batched path when its upsampling uses the default kernel sizes (8 / 7), it has at least two
// latent grids, no common randomness, and its synthesis is in the fused family.  All such jobs of a call share
//   * one launch per cascade level (all but the last), and
//   * one launch (per (cinp, C) pair) of the kernel that evaluates the last level, the synthesis and -- for the
//     full-size outputs of I frames that ask for it -- the frame tail.
// Every other job takes the per-stream path (run_synthesis), one job after the other.
bool tail_eligible(const PreparedJob &P) {
    const CcdCoolChicDesc *d = P.d;
    const int nl = P.nl;
    if (d->ups_k != 8 || d->ups_pre_k != 7 || d->common_randomness) return false;
    if (nl < 2 || nl > 16 || nl != d->syn_in) return false;
    const SynNet N = syn_net(P, nullptr);
    if (!ccd_syn_fused_family(nl, N.layers, d->n_syn_layers, d->syn_stab ? &N.stab : nullptr, N.ot)) return false;
    for (int i = 0; i + 1 < nl; i++) {
        const int gt = P.gl[i], gc = P.gl[i + 1];
        if (d->grid_h[gt] > 2 * d->grid_h[gc] || d->grid_w[gt] > 2 * d->grid_w[gc]) return false;  // (reported by the per-stream path)
    }
    return true;
}

struct TailScratch {
    size_t p = 0, q = 0, raw = 0, total = 0;
};
TailScratch tail_scratch_plan(const PreparedJob &P) {
    const CcdCoolChicDesc *d = P.d;
    TailScratch T;
    const int nl = P.nl;
    size_t o = 0;
    if (nl >= 3) {
        const int g1 = P.gl[1];
        T.p = o;
        o += al((size_t)(nl - 1) * d->grid_h[g1] * d->grid_w[g1] * 4);
    }
    if (nl >= 4) {
        const int g2 = P.gl[2];
        T.q = o;
        o += al((size_t)(nl - 2) * d->grid_h[g2] * d->grid_w[g2] * 4);
    }
    const int g0 = P.gl[0];
    if (P.resized) {
        T.raw = o;
        o += al((size_t)P.tail_C * d->grid_h[g0] * d->grid_w[g0] * 4);
    }
    T.total = o;
    return T;
}

// The float tail of one call: which path each job takes, the scratch of both paths, the job arrays in the upload
// arena and the batched path's launches.
struct TailPlan {
    struct LevelLaunch { size_t first; int count, planes, max_tw, max_th; };
    struct SynGroup { int cinp, C, n3_max, hid_max, max_w, max_h, first, count; };
    std::vector<int> order;                     // jobs of the batched path sorted by (cinp, C), one TailSynJob each
    std::vector<SynGroup> groups;               // one k_tail_syn launch each
    std::vector<std::pair<int, int>> lvl_jobs;  // (job, level) of every UpsLevelJob
    std::vector<LevelLaunch> levels;            // the batched path's k_ups_level_b launches
    size_t scratch_syn = 0, scratch_tail = 0;   // per-stream path (reused job after job), batched path
    size_t scratch_fin = 0;                     // raw output for finish_job (jobs finished one after the other)
    size_t off_syn = 0, off_lvl = 0;            // job arrays in the upload arena
    unsigned char *d_scr_syn = nullptr, *d_scr_tail = nullptr;  // the scratch of both paths (reserve_tail_scratch)
    float *d_fin = nullptr;
};

// Plans the float tail of the prepared jobs and lays out its job arrays in the call's arena A
void plan_tail(std::vector<PreparedJob> &P, const CcdJob *jobs, TailPlan &T, Arena &A) {
    for (int i = 0; i < (int)P.size(); i++) {
        PreparedJob &J = P[(size_t)i];
        J.tail = tail_eligible(J);
        if (J.tail) {
            J.tail_cinp = J.nl <= 4 ? 4 : (J.nl <= 8 ? 8 : 16);
            J.tail_C = J.d->syn_out[1];
            const TailScratch S = tail_scratch_plan(J);
            J.off_tailP = T.scratch_tail + S.p;
            J.off_tailQ = T.scratch_tail + S.q;
            J.off_tailRaw = T.scratch_tail + S.raw;
            T.scratch_tail += al(S.total);
            T.order.push_back(i);
        } else {
            T.scratch_syn = std::max(T.scratch_syn, synthesis_scratch_bytes(J.d));
        }
        if (jobs[i].finish_bitdepth != 0 && (!J.tail || J.resized))
            T.scratch_fin = std::max(T.scratch_fin, al((size_t)3 * J.d->img_h * J.d->img_w * 4));
    }
    std::stable_sort(T.order.begin(), T.order.end(), [&](int a, int b) {
        const PreparedJob &A = P[(size_t)a], &B = P[(size_t)b];
        return A.tail_cinp * 8 + A.tail_C < B.tail_cinp * 8 + B.tail_C;
    });
    // batched path: cascade level idx of every job that has one in one launch (planes = idx + 2)
    int max_levels = 0;
    for (int i : T.order) max_levels = std::max(max_levels, P[(size_t)i].nl - 2);
    for (int idx = 0; idx < max_levels; idx++) {
        TailPlan::LevelLaunch LL{T.lvl_jobs.size(), 0, idx + 2, 0, 0};
        for (int i : T.order) {
            const PreparedJob &J = P[(size_t)i];
            if (idx >= J.nl - 2) continue;
            const int gt = J.gl[J.nl - 2 - idx];
            T.lvl_jobs.push_back({i, idx});
            LL.count++;
            LL.max_tw = std::max(LL.max_tw, J.d->grid_w[gt]);
            LL.max_th = std::max(LL.max_th, J.d->grid_h[gt]);
        }
        if (LL.count) T.levels.push_back(LL);
    }
    // batched path: last level + synthesis (+ frame tail), one launch per (cinp, C)
    for (size_t t = 0; t < T.order.size(); t++) {
        const PreparedJob &J = P[(size_t)T.order[t]];
        const CcdCoolChicDesc *d = J.d;
        if (T.groups.empty() || T.groups.back().cinp != J.tail_cinp || T.groups.back().C != J.tail_C)
            T.groups.push_back(TailPlan::SynGroup{J.tail_cinp, J.tail_C, 0, 0, 0, 0, (int)t, 0});
        TailPlan::SynGroup &G = T.groups.back();
        G.count++;
        G.n3_max = std::max(G.n3_max, d->n_syn_layers - 2);
        G.hid_max = std::max(G.hid_max, d->syn_out[0]);
        G.max_w = std::max(G.max_w, d->grid_w[J.gl[0]]);
        G.max_h = std::max(G.max_h, d->grid_h[J.gl[0]]);
    }
    T.off_syn = A.take(T.order.size() * ccd_tail_job_bytes());
    T.off_lvl = A.take(T.lvl_jobs.size() * ccd_tail_level_job_bytes());
}

// Reserves the context's scratch: `before` bytes for the caller, then the float tail's (T.d_scr_syn, d_scr_tail, d_fin)
int reserve_tail_scratch(CcdContext *ctx, size_t before, TailPlan &T) {
    if (int rc = ensure_dev(ctx->scratch, before + al(T.scratch_syn) + T.scratch_tail + T.scratch_fin + 4096)) return rc;
    T.d_scr_syn = ctx->scratch.p + before;
    T.d_scr_tail = T.d_scr_syn + al(T.scratch_syn);
    T.d_fin = reinterpret_cast<float *>(T.d_scr_tail + T.scratch_tail);
    return CCD_OK;
}

// Fills the batched path's job arrays at h (host side of the upload arena dv); every grid is read at J.lat.
void fill_tail(const TailPlan &T, const std::vector<PreparedJob> &P, const CcdJob *jobs, unsigned char *h,
               const unsigned char *dv) {
    const size_t lb = ccd_tail_level_job_bytes(), jb = ccd_tail_job_bytes();
    unsigned char *d_scr_tail = T.d_scr_tail;
    for (size_t k = 0; k < T.lvl_jobs.size(); k++) {
        const int i = T.lvl_jobs[k].first, idx = T.lvl_jobs[k].second;
        const PreparedJob &J = P[(size_t)i];
        const CcdCoolChicDesc *d = J.d;
        const int gt = J.gl[J.nl - 2 - idx], gc = J.gl[J.nl - 1 - idx];
        // level idx writes P when (nl - 3 - idx) is even (the last one, idx = nl - 3, always writes P); level 0 reads
        // the coarsest int8 grid itself
        const bool to_p = ((J.nl - 3 - idx) & 1) == 0;
        float *out = reinterpret_cast<float *>(d_scr_tail + (to_p ? J.off_tailP : J.off_tailQ));
        const float *in = reinterpret_cast<const float *>(d_scr_tail + (to_p ? J.off_tailQ : J.off_tailP));
        float full_t[16], full_c[16];
        level_taps(J, idx, full_t, full_c);
        ccd_tail_fill_level(h + T.off_lvl + k * lb, J.lat[gt], idx == 0 ? nullptr : in, idx == 0 ? J.lat[gc] : nullptr,
                            out, idx + 1, d->grid_h[gc], d->grid_w[gc],
                            d->grid_h[gt], d->grid_w[gt], full_t, full_c);
    }
    for (size_t t = 0; t < T.order.size(); t++) {
        const int i = T.order[t];
        const PreparedJob &J = P[(size_t)i];
        const CcdCoolChicDesc *d = J.d;
        const int nl = J.nl, g0 = J.gl[0], g1 = J.gl[1], C = J.tail_C;
        const SynNet N = syn_net(J, reinterpret_cast<const float *>(dv + J.off_syn));
        CcdTailSynDesc S;
        memset(&S, 0, sizeof(S));
        S.lat = J.lat[g0];
        if (nl == 2) S.stk8 = J.lat[g1];
        else S.stk = reinterpret_cast<const float *>(d_scr_tail + J.off_tailP);
        S.h = d->grid_h[g0]; S.w = d->grid_w[g0]; S.ch = d->grid_h[g1]; S.cw = d->grid_w[g1]; S.cin = nl;
        S.layers = N.layers; S.n_layers = d->n_syn_layers; S.stab = d->syn_stab ? &N.stab : nullptr;
        S.ot = N.ot;
        const size_t plane = (size_t)S.h * S.w;
        const CcdJob &job = jobs[i];
        if (J.resized) {
            float *raw = reinterpret_cast<float *>(d_scr_tail + J.off_tailRaw);
            for (int c = 0; c < C; c++) S.out[c] = raw + (size_t)c * plane;
        } else if (job.finish_bitdepth != 0 && job.finish_type == 1) {
            S.out[0] = job.d_out; S.out[1] = job.d_out_u; S.out[2] = job.d_out_v;
            S.finish = 2;
        } else {
            for (int c = 0; c < C; c++) S.out[c] = job.d_out + (size_t)c * plane;
            S.finish = job.finish_bitdepth != 0 ? 1 : 0;
        }
        S.M = job.finish_bitdepth != 0 ? (float)((1 << job.finish_bitdepth) - 1) : 0.0f;
        float full_t[16], full_c[16];
        level_taps(J, nl - 2, full_t, full_c);
        S.wt1d = full_t; S.wc1d = full_c;
        S.allow_tma = J.pad_lat ? 1 : 0;
        ccd_tail_fill_syn(h + T.off_syn + t * jb, S);
    }
}

// The batched path's launches: every cascade level, then the last level + synthesis (+ frame tail) per group, then
// the final resize of the outputs computed at a smaller size than the image (motion fields, reduced-resolution I
// frames), followed by the frame tail of those that ask for it.
int launch_tail(const TailPlan &T, const std::vector<PreparedJob> &P, const CcdJob *jobs, const unsigned char *dv,
                cudaStream_t st) {
    const size_t lb = ccd_tail_level_job_bytes(), jb = ccd_tail_job_bytes();
    const unsigned char *d_scr_tail = T.d_scr_tail;
    float *d_fin = T.d_fin;
    for (const TailPlan::LevelLaunch &LL : T.levels)
        if (ccd_tail_launch_level(dv + T.off_lvl + LL.first * lb, LL.count, LL.planes, LL.max_tw, LL.max_th, st))
            return fail(CCD_ERR_CUDA, "cascade level launch failed");
    for (const TailPlan::SynGroup &G : T.groups) {
        const int e = ccd_tail_launch_syn(dv + T.off_syn + (size_t)G.first * jb, G.count, G.cinp, G.C, G.n3_max, G.hid_max,
                                          G.max_w, G.max_h, st);
        if (e != 0) return fail(CCD_ERR_CUDA, "fused tail launch failed (%d)", e);
    }
    for (int i : T.order) {
        const PreparedJob &J = P[(size_t)i];
        if (!J.resized) continue;
        const CcdCoolChicDesc *d = J.d;
        float *out = jobs[i].finish_bitdepth != 0 ? d_fin : jobs[i].d_out;
        int rc = resize_output(d, reinterpret_cast<const float *>(d_scr_tail + J.off_tailRaw), J.tail_C,
                               d->grid_h[J.gl[0]], d->grid_w[J.gl[0]], out, st);
        if (!rc) rc = finish_job(jobs[i], out, st);
        if (rc) return rc;
    }
    return CCD_OK;
}

// The float tail of a call (DESIGN §4.2) once its job arrays are on the device at dv: the batched path's launches,
// then every other job, one after the other, through the per-stream path.  A failing job gets its status.
int run_tail(const TailPlan &T, const std::vector<PreparedJob> &P, CcdJob *jobs, const unsigned char *dv, cudaStream_t st) {
    if (int rc = launch_tail(T, P, jobs, dv, st)) return rc;
    for (int i = 0; i < (int)P.size(); i++) {
        const PreparedJob &J = P[(size_t)i];
        if (J.tail) continue;
        float *out = jobs[i].finish_bitdepth != 0 ? T.d_fin : jobs[i].d_out;
        int rc = run_synthesis(J, reinterpret_cast<const float *>(dv + J.off_syn), out, T.d_scr_syn, T.scratch_syn, st);
        if (!rc) rc = finish_job(jobs[i], out, st);
        if (rc) {
            jobs[i].status = rc;
            return rc;
        }
    }
    return CCD_OK;
}

// A zeroed device region of at least `bytes` in the context.  A region whose clear could not be queued is given back,
// so that no later call takes it for zeros.
int ensure_zeros(CcdContext *ctx, size_t bytes, cudaStream_t st) {
    if (bytes <= ctx->zeros.cap) return CCD_OK;
    if (int rc = ensure_dev(ctx->zeros, bytes)) return rc;
    const cudaError_t e = cudaMemsetAsync(ctx->zeros.p, 0, ctx->zeros.cap, st);
    if (e == cudaSuccess) return CCD_OK;
    cudaFree(ctx->zeros.p);
    ctx->zeros.p = nullptr;
    ctx->zeros.cap = 0;
    return fail(CCD_ERR_CUDA, "clearing the zero region failed: %s", cudaGetErrorString(e));
}

}  // namespace

// =========================================================================================
extern "C" {

int ccd_version(void) { return CCD_VERSION; }
int ccd_sizeof_desc(void) { return (int)sizeof(CcdCoolChicDesc); }
const char *ccd_last_error(const CcdContext *) { return g_err.c_str(); }

int ccd_create(int device_ordinal, CcdContext **out) {
    if (!out) return fail(CCD_ERR_ARG, "null out pointer");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(CCD_ERR_NO_DEVICE, "no CUDA device available (%s): libccdec has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (device_ordinal < 0 || device_ordinal >= n) return fail(CCD_ERR_ARG, "device %d out of range [0,%d)", device_ordinal, n);
    CUDA_TRY(cudaSetDevice(device_ordinal));
    CcdContext *c = new CcdContext();
    c->device = device_ordinal;
    {
        int nsm = 0;
        if (cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device_ordinal) == cudaSuccess && nsm > 0) c->n_sm = nsm;
    }
    int rc = CCD_OK;
    do {
        if (cudaMalloc(&c->d_scale, CCD_N_SCALE * 4) != cudaSuccess ||
            cudaMalloc(&c->d_cdf, (size_t)CCD_N_SCALE * 256 * CCD_WIN * 4) != cudaSuccess) {
            rc = fail(CCD_ERR_NOMEM, "cudaMalloc of the cumulative table failed");
            break;
        }
        if (cudaMemcpy(c->d_scale, k_scale_bits, CCD_N_SCALE * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
            rc = fail(CCD_ERR_CUDA, "scale table upload failed");
            break;
        }
        int ce = ccd_cdf_table_build(c->d_cdf, c->d_scale, 0);
        if (ce == 0) ce = (int)cudaDeviceSynchronize();
        if (ce != 0) {
            rc = fail(CCD_ERR_CUDA, "cumulative table kernel failed: %s", cudaGetErrorString((cudaError_t)ce));
            break;
        }
        for (int i = 0; i < 4; i++)
            if (cudaEventCreate(&c->ev[i]) != cudaSuccess) rc = fail(CCD_ERR_CUDA, "event creation failed");
    } while (0);
    if (rc) {
        ccd_destroy(c);
        return rc;
    }
    *out = c;
    return CCD_OK;
}

void ccd_destroy(CcdContext *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->d_scale) cudaFree(c->d_scale);
    if (c->d_cdf) cudaFree(c->d_cdf);
    if (c->upload.p) cudaFree(c->upload.p);
    if (c->scratch.p) cudaFree(c->scratch.p);
    if (c->zeros.p) cudaFree(c->zeros.p);
    if (c->h_pin) cudaFreeHost(c->h_pin);
    for (int i = 0; i < 4; i++)
        if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    for (int i = 0; i < 3; i++) {
        if (c->aux[i]) cudaStreamDestroy(c->aux[i]);
        if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]);
    }
    delete c;
}

int64_t ccd_nn_count(const CcdCoolChicDesc *desc) {
    NNLayout L;
    int rc = nn_layout(desc, &L);
    return rc ? rc : L.total;
}

int64_t ccd_latent_count(const CcdCoolChicDesc *d, int64_t offsets_by_grid[CCD_MAX_GRIDS]) {
    int rc = validate_desc(d);
    if (rc) return rc;
    int64_t off = 0;
    for (int g = d->n_grids - 1; g >= 0; g--) {
        if (offsets_by_grid) offsets_by_grid[g] = off;
        off += (int64_t)d->grid_h[g] * d->grid_w[g];
    }
    return off;
}

int64_t ccd_decode_nn(const CcdCoolChicDesc *desc, const uint8_t *nn_bytes, size_t nn_nbytes, int64_t *out_ints,
                      size_t cap) {
    NNLayout L;
    int rc = nn_layout(desc, &L);
    if (rc) return rc;
    if (!nn_bytes || !out_ints || (size_t)L.total > cap) return fail(CCD_ERR_ARG, "bad buffer");
    return decode_nn_host(desc, L, nn_bytes, nn_nbytes, out_ints);
}

// The entropy stage of every job, then (tail) its float tail: upsampling, synthesis and the frame tail it asks for.
static int decode_impl_body(CcdContext *ctx, CcdJob *jobs, int n_jobs, const int64_t *const *nn_ints, bool tail,
                            int mode, uint64_t seed, uint32_t *const *d_out_words, int64_t out_cap,
                            int32_t (*statuses)[16], cudaStream_t st) {
    if (tail)
        for (int i = 0; i < n_jobs; i++)
            if (!jobs[i].d_out) return fail(CCD_ERR_ARG, "job %d: null output pointer", i);
    CUDA_TRY(cudaEventRecord(ctx->ev[0], st));

    std::vector<PreparedJob> P((size_t)n_jobs);
    Arena A;
    size_t scratch_lat = 0;
    for (int i = 0; i < n_jobs; i++) {
        P[(size_t)i].job = &jobs[i];
        P[(size_t)i].d = jobs[i].desc;
        const bool own_lat = !jobs[i].d_latents;
        P[(size_t)i].pad_lat = own_lat && mode == 0;
        int rc = prepare_job(P[(size_t)i], nn_ints ? nn_ints[i] : nullptr);
        PreparedJob &J = P[(size_t)i];
        if (!rc) rc = entropy_smem_ok(J.smem);
        if (rc) {
            jobs[i].status = rc;
            return rc;
        }
        if (mode == 0 && (!jobs[i].latent_bytes && jobs[i].latent_nbytes))
            return fail(CCD_ERR_ARG, "job %d: null latent bytes", i);
        const size_t nwords = mode == 0 ? jobs[i].latent_nbytes / 4 : 0;
        J.off_words = A.take(nwords * 4 + 16);
        J.off_blob = A.take(J.blob.size());
        J.off_syn = A.take(J.syn_f.size() * 4);
        if (tail && (rc = check_finish(jobs[i], J, i))) return rc;
        J.off_lat = scratch_lat;
        if (own_lat) scratch_lat += al((size_t)J.lat_bytes);
    }
    // the float tail's device-resident job arrays (filled below, uploaded with everything else)
    TailPlan T;
    if (tail) plan_tail(P, jobs, T, A);
    const size_t off_streams = A.take(sizeof(EntStream) * (size_t)n_jobs);
    const size_t off_status = A.take(sizeof(int32_t[16]) * (size_t)n_jobs);  // results: zeroed status words per job
    int rc;
    if ((rc = stage(ctx, A))) return rc;
    unsigned char *h = A.h, *dv = A.dv;
    if ((rc = reserve_tail_scratch(ctx, scratch_lat, T))) return rc;

    // group jobs by kernel configuration so that each group is one launch
    std::vector<int> order((size_t)n_jobs);
    for (int i = 0; i < n_jobs; i++) order[(size_t)i] = i;
    auto key = [&](int i) {
        const PreparedJob &J = P[(size_t)i];
        return J.fast ? (J.d->n_ctx * 64 + J.d->n_ifce_out) : -1;
    };
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key(a) < key(b); });

    for (int i = 0; i < n_jobs; i++) {
        PreparedJob &J = P[(size_t)i];
        const size_t nbytes4 = mode == 0 ? jobs[i].latent_nbytes / 4 * 4 : 0;
        memset(h + J.off_words, 0, al(nbytes4 + 16));
        if (nbytes4) memcpy(h + J.off_words, jobs[i].latent_bytes, nbytes4);
        memcpy(h + J.off_blob, J.blob.data(), J.blob.size());
        if (!J.syn_f.empty()) memcpy(h + J.off_syn, J.syn_f.data(), J.syn_f.size() * 4);
        int8_t *lat = jobs[i].d_latents;
        if (!lat) lat = reinterpret_cast<int8_t *>(ctx->scratch.p + J.off_lat);
        for (int g = 0; g < J.d->n_grids; g++) J.lat[g] = lat + J.lat_off_by_grid[g];
        EntStream &S = J.es;
        S.mode = mode;
        S.prod_mask = ctx->prod_mask;
        S.seed = seed + (uint64_t)i;
        S.words = reinterpret_cast<const uint32_t *>(dv + J.off_words);
        S.n_words = (int64_t)(nbytes4 / 4);
        S.latents = lat;
        S.blob = dv + J.off_blob;
        S.status = reinterpret_cast<int32_t *>(dv + off_status) + 16 * (size_t)i;
        S.out_words = d_out_words ? d_out_words[i] : nullptr;
        S.out_cap = d_out_words ? out_cap : 0;
    }
    for (int t = 0; t < n_jobs; t++)
        memcpy(h + off_streams + sizeof(EntStream) * (size_t)t, &P[(size_t)order[(size_t)t]].es, sizeof(EntStream));
    memset(h + off_status, 0, A.end - off_status);

    if (tail) fill_tail(T, P, jobs, h, dv);
    CUDA_TRY(cudaMemcpyAsync(dv, h, A.end, cudaMemcpyHostToDevice, st));
    ctx->last_upload_bytes = A.end;
    CUDA_TRY(cudaEventRecord(ctx->ev[1], st));

    int t = 0, g = 0;
    while (t < n_jobs) {
        int u = t;
        size_t smem = 0;
        while (u < n_jobs && key(order[(size_t)u]) == key(order[(size_t)t])) {
            smem = std::max(smem, P[(size_t)order[(size_t)u]].smem);
            u++;
        }
        const PreparedJob &J0 = P[(size_t)order[(size_t)t]];
        // more streams than SMs: 8-warp CTAs, two per SM (registers: 2 x 256 x 128; shared memory permitting)
        const bool narrow = mode == 0 && (u - t) > ctx->n_sm &&
                            2 * (smem + 1024) <= (size_t)CCD_SMEM_MAX;
        EntLaunchCfg cfg{J0.d->n_ctx, J0.d->flag_ifce ? J0.d->n_ifce_out : 0, J0.fast, smem,
                         narrow ? CCD_ENT_THREADS_NARROW : CCD_ENT_THREADS};
        // group 0 on the caller's stream, the next ones on auxiliary streams forked after the upload
        cudaStream_t sg = st;
        if (g > 0) {
            const int a = (g - 1) % 3;
            if (!ctx->aux[a]) {
                CUDA_TRY(cudaStreamCreateWithFlags(&ctx->aux[a], cudaStreamNonBlocking));
                CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_join[a], cudaEventDisableTiming));
            }
            sg = ctx->aux[a];
            CUDA_TRY(cudaStreamWaitEvent(sg, ctx->ev[1], 0));  // the upload (recorded on st before any launch)
        }
        int e = ccd_entropy_launch(reinterpret_cast<const EntStream *>(dv + off_streams) + t, u - t, cfg, ctx->d_cdf,
                                   ctx->d_scale, sg);
        if (e != 0) return fail(CCD_ERR_CUDA, "entropy kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
        if (g > 0) {
            const int a = (g - 1) % 3;
            CUDA_TRY(cudaEventRecord(ctx->ev_join[a], sg));
            CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join[a], 0));
        }
        t = u;
        g++;
    }
    CUDA_TRY(cudaEventRecord(ctx->ev[2], st));
    if (tail && (rc = run_tail(T, P, jobs, dv, st))) return rc;
    CUDA_TRY(cudaEventRecord(ctx->ev[3], st));
    if ((rc = download(A, off_status, st, "kernel"))) return rc;
    cudaEventElapsedTime(&ctx->last_ms[2], ctx->ev[0], ctx->ev[1]);
    cudaEventElapsedTime(&ctx->last_ms[0], ctx->ev[1], ctx->ev[2]);
    cudaEventElapsedTime(&ctx->last_ms[1], ctx->ev[2], ctx->ev[3]);
    const auto *words = reinterpret_cast<const int32_t(*)[16]>(h + off_status);
    if (statuses) memcpy(statuses, words, sizeof(int32_t[16]) * (size_t)n_jobs);
    memcpy(ctx->last_status, words[n_jobs - 1], sizeof(int32_t[16]));
    return report(jobs, n_jobs, words, [&](int i) {
        return fail(jobs[i].status, "job %d: corrupt latent payload (range decoder desynchronised)", i);
    });
}

static int decode_impl(CcdContext *ctx, CcdJob *jobs, int n_jobs, const int64_t *const *nn_ints, bool tail, int mode,
                       uint64_t seed, uint32_t *const *d_out_words, int64_t out_cap, int32_t (*statuses)[16],
                       void *cuda_stream) {
    return job_call(ctx, jobs, n_jobs, cuda_stream, [&](cudaStream_t st) -> int {
        return decode_impl_body(ctx, jobs, n_jobs, nn_ints, tail, mode, seed, d_out_words, out_cap, statuses, st);
    });
}

int ccd_decode_many(CcdContext *ctx, CcdJob *jobs, int n_jobs, void *cuda_stream) {
    return decode_impl(ctx, jobs, n_jobs, nullptr, true, 0, 0, nullptr, 0, nullptr, cuda_stream);
}

int ccd_decode_coolchic(CcdContext *ctx, const CcdCoolChicDesc *desc, const uint8_t *nn_bytes, size_t nn_nbytes,
                        const uint8_t *latent_bytes, size_t latent_nbytes, float *d_out, int8_t *d_latents,
                        void *cuda_stream) {
    CcdJob j{desc, nn_bytes, nn_nbytes, latent_bytes, latent_nbytes, d_out, d_latents, 0, 0, 0, nullptr, nullptr};
    return ccd_decode_many(ctx, &j, 1, cuda_stream);
}

int ccd_decode_latents(CcdContext *ctx, const CcdCoolChicDesc *desc, const int64_t *nn_ints, const uint8_t *latent_bytes,
                       size_t latent_nbytes, int8_t *d_latents, void *cuda_stream) {
    if (!d_latents || !nn_ints) return fail(CCD_ERR_ARG, "null pointer");
    CcdJob j{desc, nullptr, 0, latent_bytes, latent_nbytes, nullptr, d_latents, 0, 0, 0, nullptr, nullptr};
    const int64_t *nn[1] = {nn_ints};
    return decode_impl(ctx, &j, 1, nn, false, 0, 0, nullptr, 0, nullptr, cuda_stream);
}

int ccd_encode_latents(CcdContext *ctx, const CcdCoolChicDesc *desc, const int64_t *nn_ints, int mode, uint64_t seed,
                       int8_t *d_latents, uint32_t *d_out_words, int64_t out_cap_words, int64_t *n_words_out,
                       int32_t *slow_out, void *cuda_stream) {
    if (!d_latents || !nn_ints || !d_out_words || (mode != 1 && mode != 2)) return fail(CCD_ERR_ARG, "bad argument");
    CcdJob j{desc, nullptr, 0, nullptr, 0, nullptr, d_latents, 0, 0, 0, nullptr, nullptr};
    const int64_t *nn[1] = {nn_ints};
    uint32_t *ow[1] = {d_out_words};
    int32_t stt[1][16];
    int rc = decode_impl(ctx, &j, 1, nn, false, mode, seed, ow, out_cap_words, stt, cuda_stream);
    if (rc) return rc;
    if (n_words_out) *n_words_out = stt[0][3];
    if (slow_out) *slow_out = stt[0][2];
    if (stt[0][3] > out_cap_words) return fail(CCD_ERR_ARG, "output buffer too small (%d words needed)", stt[0][3]);
    return CCD_OK;
}

// The float tail of every job on the caller's latents: decode's plan, arrays and launches, no entropy stage.  A grid
// the job masks is read from the context's zeroed region instead of its latents.
static int synthesize_body(CcdContext *ctx, CcdSynthJob *jobs, int n_jobs, cudaStream_t st) {
    std::vector<PreparedJob> P((size_t)n_jobs);
    std::vector<CcdJob> tj((size_t)n_jobs);  // each job's outputs and frame-tail request, as the float tail takes them
    Arena A;
    size_t max_grid = 16;
    for (int i = 0; i < n_jobs; i++) {
        CcdSynthJob &S = jobs[i];
        if (!S.desc || !S.nn_ints) return S.status = fail(CCD_ERR_ARG, "job %d: null descriptor or network integers", i);
        if (!S.d_latents || !S.d_out) return S.status = fail(CCD_ERR_ARG, "job %d: null latents or output pointer", i);
        tj[(size_t)i] = CcdJob{S.desc, nullptr, 0, nullptr, 0, S.d_out, nullptr, CCD_OK, S.finish_bitdepth, S.finish_type,
                               S.d_out_u, S.d_out_v};
        PreparedJob &J = P[(size_t)i];
        J.job = &tj[(size_t)i];
        J.d = S.desc;
        if (int rc = prepare_synthesis(J, S.nn_ints)) return S.status = rc;
        const CcdCoolChicDesc *d = J.d;
        for (int g = 0; g < 32; g++) {
            if (!((S.zero_grids >> g) & 1u)) continue;
            if (g >= d->n_grids)
                return S.status = fail(CCD_ERR_ARG, "job %d: zero_grids bit %d, the stream has %d grids", i, g, d->n_grids);
            if (d->grid_is_hyper[g])
                return S.status = fail(CCD_ERR_ARG, "job %d: zero_grids bit %d is a hyperlatent grid, which no synthesis reads", i, g);
        }
        if (int rc = check_finish(tj[(size_t)i], J, i)) return S.status = rc;
        J.off_syn = A.take(J.syn_f.size() * 4);
        for (int g = 0; g < d->n_grids; g++) max_grid = std::max(max_grid, (size_t)d->grid_h[g] * d->grid_w[g]);
    }
    TailPlan T;
    plan_tail(P, tj.data(), T, A);
    // results: one status word per job, zero on the way up.  No float-tail kernel reports a per-job fault, so the download
    // is the call's synchronisation and the report every job call makes.
    const size_t off_status = A.take(sizeof(int32_t) * (size_t)n_jobs);
    if (int rc = stage(ctx, A)) return rc;
    if (int rc = reserve_tail_scratch(ctx, 0, T)) return rc;
    if (int rc = ensure_zeros(ctx, max_grid, st)) return rc;
    for (int i = 0; i < n_jobs; i++) {
        PreparedJob &J = P[(size_t)i];
        if (!J.syn_f.empty()) memcpy(A.h + J.off_syn, J.syn_f.data(), J.syn_f.size() * 4);
        for (int g = 0; g < J.d->n_grids; g++)
            J.lat[g] = ((jobs[i].zero_grids >> g) & 1u) ? reinterpret_cast<const int8_t *>(ctx->zeros.p)
                                                        : jobs[i].d_latents + J.lat_off_by_grid[g];
    }
    memset(A.h + off_status, 0, A.end - off_status);
    fill_tail(T, P, tj.data(), A.h, A.dv);
    CUDA_TRY(cudaMemcpyAsync(A.dv, A.h, A.end, cudaMemcpyHostToDevice, st));
    if (int rc = run_tail(T, P, tj.data(), A.dv, st)) {
        for (int i = 0; i < n_jobs; i++)
            if (tj[(size_t)i].status != CCD_OK) jobs[i].status = tj[(size_t)i].status;
        return rc;
    }
    if (int rc = download(A, off_status, st, "synthesis")) return rc;
    return report(jobs, n_jobs, reinterpret_cast<const int32_t *>(A.h + off_status),
                  [&](int i) { return fail(jobs[i].status, "job %d: synthesis failed", i); });
}

int ccd_synthesize_many(CcdContext *ctx, CcdSynthJob *jobs, int n_jobs, void *cuda_stream) {
    return job_call(ctx, jobs, n_jobs, cuda_stream, [&](cudaStream_t st) -> int { return synthesize_body(ctx, jobs, n_jobs, st); });
}

static int latent_rate_body(CcdContext *ctx, CcdRateJob *jobs, int n_jobs, cudaStream_t st) {
    std::vector<PreparedJob> P((size_t)n_jobs);
    std::vector<RateTile> tiles;
    // tiles of job i, decode-order grid gi: [tile_at[i][gi], tile_at[i][gi + 1])
    std::vector<std::vector<size_t>> tile_at((size_t)n_jobs);
    std::vector<RateSpatialDev> sp;
    int64_t max_pixels = 0;
    Arena A;
    size_t smem = 0;
    for (int i = 0; i < n_jobs; i++) {
        CcdRateJob &R = jobs[i];
        R.bad_index = -1;
        if (!R.desc || !R.nn_ints || !R.d_latents || !R.d_bits) return R.status = fail(CCD_ERR_ARG, "job %d: null pointer", i);
        PreparedJob &J = P[(size_t)i];
        J.d = R.desc;
        int rc = prepare_job(J, R.nn_ints);  // the decoder's build_arm / pack_arm / pack_ifce and fast-path choice
        if (rc) return R.status = rc;
        J.off_blob = A.take(J.blob.size());
        smem = std::max(smem, ccd_rate_smem_bytes(J.es.arm_blob_bytes, J.es.ifce_blob_max));
        const CcdCoolChicDesc *d = J.d;
        tile_at[(size_t)i].push_back(tiles.size());
        for (int gi = 0; gi < d->n_grids; gi++) {
            const EntGrid &G = J.es.grid[gi];
            for (int y0 = 0; y0 < G.h; y0 += CCD_RATE_TH)
                for (int x0 = 0; x0 < G.w; x0 += CCD_RATE_TW) tiles.push_back(RateTile{i, gi, y0, x0});
            tile_at[(size_t)i].push_back(tiles.size());
        }
        if (R.d_spatial) {
            RateSpatialDev S;
            memset(&S, 0, sizeof(S));
            S.bits = R.d_bits;
            S.out = R.d_spatial;
            S.H = d->img_h;
            S.W = d->img_w;
            S.n_grids = d->n_grids;
            for (int g = 0; g < d->n_grids; g++) {
                S.h[g] = d->grid_h[g];
                S.w[g] = d->grid_w[g];
                S.off[g] = J.lat_off_by_grid[g];
                S.ratio[g] = (float)(((double)d->img_h * d->img_w) / ((double)d->grid_h[g] * d->grid_w[g]));
                S.sy[g] = (float)d->grid_h[g] / (float)d->img_h;
                S.sx[g] = (float)d->grid_w[g] / (float)d->img_w;
            }
            sp.push_back(S);
            max_pixels = std::max(max_pixels, (int64_t)d->img_h * d->img_w);
        }
    }
    if (tiles.size() > (size_t)INT32_MAX) return fail(CCD_ERR_UNSUPPORTED, "too many rate tiles");
    if (smem > CCD_SMEM_MAX) return fail(CCD_ERR_UNSUPPORTED, "rate pass needs %zu bytes of shared memory", smem);
    const size_t off_es = A.take(sizeof(EntStream) * (size_t)n_jobs);
    const size_t off_jobs = A.take(sizeof(RateJobDev) * (size_t)n_jobs);
    const size_t off_tiles = A.take(sizeof(RateTile) * tiles.size());
    const size_t off_sp = A.take(sizeof(RateSpatialDev) * sp.size());
    // results: the bad words (~0 before the launch), then the partials, which are not uploaded
    const size_t off_bad = A.take(sizeof(unsigned long long) * (size_t)n_jobs);
    const size_t off_part = A.take(sizeof(double) * tiles.size());
    if (int rc = stage(ctx, A)) return rc;
    memset(A.h + off_bad, 0xff, sizeof(unsigned long long) * (size_t)n_jobs);
    for (int i = 0; i < n_jobs; i++) {
        PreparedJob &J = P[(size_t)i];
        memcpy(A.h + J.off_blob, J.blob.data(), J.blob.size());
        J.es.latents = const_cast<int8_t *>(jobs[i].d_latents);
        J.es.blob = A.dv + J.off_blob;
        memcpy(A.h + off_es + sizeof(EntStream) * (size_t)i, &J.es, sizeof(EntStream));
        RateJobDev D;
        D.es = reinterpret_cast<const EntStream *>(A.dv + off_es) + i;
        D.bits = jobs[i].d_bits;
        D.freq = jobs[i].d_freq;
        D.mu_sc = jobs[i].d_mu_sc;
        D.bad = reinterpret_cast<unsigned long long *>(A.dv + off_bad) + i;
        D.kind = ccd_rate_kind(J.d->n_ctx, J.es.cf, J.fast);
        memcpy(A.h + off_jobs + sizeof(RateJobDev) * (size_t)i, &D, sizeof(D));
    }
    memcpy(A.h + off_tiles, tiles.data(), sizeof(RateTile) * tiles.size());
    if (!sp.empty()) memcpy(A.h + off_sp, sp.data(), sizeof(RateSpatialDev) * sp.size());
    CUDA_TRY(cudaMemcpyAsync(A.dv, A.h, off_part, cudaMemcpyHostToDevice, st));
    int e = ccd_rate_launch(reinterpret_cast<const RateTile *>(A.dv + off_tiles), (int)tiles.size(),
                            reinterpret_cast<const RateJobDev *>(A.dv + off_jobs), smem, ctx->d_cdf, ctx->d_scale,
                            reinterpret_cast<double *>(A.dv + off_part), st);
    if (e != 0) return fail(CCD_ERR_CUDA, "rate kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    if (!sp.empty()) {
        e = ccd_rate_spatial_launch(reinterpret_cast<const RateSpatialDev *>(A.dv + off_sp), (int)sp.size(), max_pixels, st);
        if (e != 0) return fail(CCD_ERR_CUDA, "spatial rate launch failed: %s", cudaGetErrorString((cudaError_t)e));
    }
    if (int rc = download(A, off_bad, st, "rate kernel")) return rc;
    const double *part = reinterpret_cast<const double *>(A.h + off_part);
    for (int i = 0; i < n_jobs; i++) {
        const std::vector<size_t> &at = tile_at[(size_t)i];  // a grid's sum: its tiles in order
        const int n_grids = P[(size_t)i].d->n_grids;
        for (int g = 0; g < CCD_MAX_GRIDS; g++) jobs[i].grid_bits[g] = 0.0;
        for (int gi = 0; gi < n_grids; gi++) jobs[i].grid_bits[n_grids - 1 - gi] = ordered_sum(part + at[gi], at[gi + 1] - at[gi]);
    }
    return report(jobs, n_jobs, reinterpret_cast<const unsigned long long *>(A.h + off_bad), [&](int i) {
        return fail(CCD_ERR_ARG, "job %d: latent %lld is outside [-64, 63]", i, (long long)jobs[i].bad_index);
    });
}

int ccd_latent_rate(CcdContext *ctx, CcdRateJob *jobs, int n_jobs, void *cuda_stream) {
    return job_call(ctx, jobs, n_jobs, cuda_stream, [&](cudaStream_t st) -> int { return latent_rate_body(ctx, jobs, n_jobs, st); });
}

// The checks of a job that compares a finished frame with its source samples (CcdDistJob, CcdSsimJob)
extern "C++" template <class Job>
int check_frame_job(Job &J, int i) {
    J.bad_index = -1;
    if (!J.d_planes[0] || !J.d_planes[1] || !J.d_planes[2] || !J.d_src || J.h < 1 || J.w < 1)
        return J.status = fail(CCD_ERR_ARG, "job %d: bad argument", i);
    if (J.bitdepth < 1 || J.bitdepth > 16) return J.status = fail(CCD_ERR_ARG, "job %d: bad bitdepth %d", i, J.bitdepth);
    if (J.chroma_shift < 0 || J.chroma_shift > 1 || J.src_layout < 0 || J.src_layout > 1 || (J.src_layout && J.chroma_shift))
        return J.status = fail(CCD_ERR_ARG, "job %d: bad layout", i);
    if (J.chroma_shift && ((J.h | J.w) & 1))
        return J.status = fail(CCD_ERR_ARG, "job %d: 4:2:0 needs even frame sizes, got %dx%d", i, J.h, J.w);
    if ((int64_t)J.h * J.w > (int64_t)INT32_MAX / 3) return J.status = fail(CCD_ERR_UNSUPPORTED, "job %d: frame too large", i);
    return CCD_OK;
}

// The message of a job whose decoded frame has a sample off the k / M grid (report(), after the kernel)
extern "C++" template <class Job>
int off_grid_error(const Job &J, int i) {
    return fail(CCD_ERR_ARG, "job %d: decoded sample %lld is off the k / (2^%d - 1) grid", i, (long long)J.bad_index,
                J.bitdepth);
}

static int frame_distortion_body(CcdContext *ctx, CcdDistJob *jobs, int n_jobs, cudaStream_t st) {
    int64_t max_pixels = 1;
    for (int i = 0; i < n_jobs; i++) {
        if (int rc = check_frame_job(jobs[i], i)) return rc;
        max_pixels = std::max(max_pixels, (int64_t)jobs[i].h * jobs[i].w);
    }
    if (n_jobs > 65535) return fail(CCD_ERR_UNSUPPORTED, "%d frames in one call (at most 65535)", n_jobs);
    // the job array, then the results: sse[n][3] and max_abs[n][3] zeroed, bad[n] ~0
    Arena A;
    const size_t n = (size_t)n_jobs, off_jobs = A.take(sizeof(DistJobDev) * n), off_sse = A.take(24 * n);
    const size_t off_bad = A.take(8 * n, 8), off_max = A.take(12 * n, 4);
    if (int rc = stage(ctx, A)) return rc;
    memset(A.h + off_sse, 0, A.end - off_sse);
    memset(A.h + off_bad, 0xff, 8 * n);
    for (int i = 0; i < n_jobs; i++) {
        const CcdDistJob &J = jobs[i];
        DistJobDev D;
        for (int c = 0; c < 3; c++) D.p[c] = J.d_planes[c];
        D.src = J.d_src;
        D.map = J.d_map;
        D.h = J.h;
        D.w = J.w;
        D.cs = J.chroma_shift;
        D.hwc = J.src_layout;
        const double M = (double)((1 << J.bitdepth) - 1);
        D.M = (float)M;
        D.M2 = (float)(M * M);
        D.wide = J.bitdepth > 8;
        D.sse = reinterpret_cast<unsigned long long *>(A.dv + off_sse) + 3 * i;
        D.bad = reinterpret_cast<unsigned long long *>(A.dv + off_bad) + i;
        D.max_abs = reinterpret_cast<unsigned int *>(A.dv + off_max) + 3 * i;
        memcpy(A.h + off_jobs + sizeof(DistJobDev) * (size_t)i, &D, sizeof(D));
    }
    CUDA_TRY(cudaMemcpyAsync(A.dv, A.h, A.end, cudaMemcpyHostToDevice, st));
    int e = ccd_dist_launch(reinterpret_cast<const DistJobDev *>(A.dv + off_jobs), n_jobs, max_pixels, ctx->n_sm, st);
    if (e != 0) return fail(CCD_ERR_CUDA, "frame distortion launch failed: %s", cudaGetErrorString((cudaError_t)e));
    if (int rc = download(A, off_sse, st, "frame distortion")) return rc;
    for (int i = 0; i < n_jobs; i++) {
        memcpy(jobs[i].sse, A.h + off_sse + 24 * (size_t)i, 24);
        memcpy(jobs[i].max_abs, A.h + off_max + 12 * (size_t)i, 12);
    }
    return report(jobs, n_jobs, reinterpret_cast<const unsigned long long *>(A.h + off_bad), [&](int i) { return off_grid_error(jobs[i], i); });
}

int ccd_frame_distortion(CcdContext *ctx, CcdDistJob *jobs, int n_jobs, void *cuda_stream) {
    return job_call(ctx, jobs, n_jobs, cuda_stream, [&](cudaStream_t st) -> int { return frame_distortion_body(ctx, jobs, n_jobs, st); });
}

static int frame_ssim_body(CcdContext *ctx, CcdSsimJob *jobs, int n_jobs, cudaStream_t st) {
    constexpr int S = CCD_SSIM_SCALES;
    const size_t n = (size_t)n_jobs;
    auto side = [&](int i, int c, int j, bool width) {  // plane c of job i at scale j
        const CcdSsimJob &J = jobs[i];
        return ((width ? J.w : J.h) >> (c ? J.chroma_shift : 0)) >> j;
    };
    auto tiles = [&](int i, int c, int j) { return ccd_ssim_tiles(side(i, c, j, false), side(i, c, j, true)); };
    // the job's partials at scale j start at part_at[i * S + j] (pairs, planes in order); the pyramid levels 1..4 of
    // every plane of every job, one after the other, in the context's scratch
    std::vector<size_t> part_at(n * S);
    size_t n_part = 0, pyr_bytes = 0;
    int max_tiles[S] = {0, 0, 0, 0, 0};
    for (int i = 0; i < n_jobs; i++) {
        if (int rc = check_frame_job(jobs[i], i)) return rc;
        for (int c = 0; c < 3; c++)
            if (std::min(side(i, c, 0, false), side(i, c, 0, true)) < 176)
                return jobs[i].status = fail(CCD_ERR_ARG, "job %d: plane %d is %dx%d, MS-SSIM needs both sides >= 176", i, c,
                                             side(i, c, 0, true), side(i, c, 0, false));
        for (int j = 0; j < S; j++) {
            part_at[(size_t)i * S + j] = n_part;
            const int t = tiles(i, 0, j) + tiles(i, 1, j) + tiles(i, 2, j);
            max_tiles[j] = std::max(max_tiles[j], t);
            n_part += (size_t)t;
            for (int c = 0; j > 0 && c < 3; c++) pyr_bytes += al(sizeof(uint2) * (size_t)side(i, c, j, false) * side(i, c, j, true));
        }
    }
    if (n_jobs > 65535) return fail(CCD_ERR_UNSUPPORTED, "%d frames in one call (at most 65535)", n_jobs);
    // the job array, then the results: bad[n] ~0, then the partials, which are not uploaded
    Arena A;
    const size_t off_jobs = A.take(sizeof(SsimJobDev) * n), off_bad = A.take(8 * n, 8);
    const size_t off_part = A.take(2 * sizeof(double) * n_part, 8);
    if (int rc = stage(ctx, A)) return rc;
    if (int rc = ensure_dev(ctx->scratch, pyr_bytes)) return rc;
    memset(A.h + off_bad, 0xff, 8 * n);
    double *d_part = reinterpret_cast<double *>(A.dv + off_part);
    unsigned char *pyr = ctx->scratch.p;
    for (int i = 0; i < n_jobs; i++) {
        const CcdSsimJob &J = jobs[i];
        SsimJobDev D;
        memset(&D, 0, sizeof(D));
        for (int c = 0; c < 3; c++) {
            D.p[c] = J.d_planes[c];
            D.map[c] = J.d_map[c];
        }
        for (int j = 0; j < S; j++) {
            D.part[j] = d_part + 2 * part_at[(size_t)i * S + j];
            for (int c = 0; j > 0 && c < 3; c++) {
                D.lvl[c][j] = reinterpret_cast<uint2 *>(pyr);
                pyr += al(sizeof(uint2) * (size_t)side(i, c, j, false) * side(i, c, j, true));
            }
        }
        D.src = J.d_src;
        D.h = J.h;
        D.w = J.w;
        D.cs = J.chroma_shift;
        D.hwc = J.src_layout;
        D.wide = J.bitdepth > 8;
        const double M = (double)((1 << J.bitdepth) - 1);
        D.M = (float)M;
        D.C1 = (0.01 * M) * (0.01 * M);
        D.C2 = (0.03 * M) * (0.03 * M);
        D.bad = reinterpret_cast<unsigned long long *>(A.dv + off_bad) + i;
        memcpy(A.h + off_jobs + sizeof(SsimJobDev) * (size_t)i, &D, sizeof(D));
    }
    double g[11], gs = 0.0;  // the Gaussian window, sigma 1.5, normalised to sum 1
    for (int k = 0; k < 11; k++) gs += (g[k] = std::exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)));
    for (int k = 0; k < 11; k++) g[k] /= gs;
    CUDA_TRY(cudaMemcpyAsync(A.dv, A.h, off_part, cudaMemcpyHostToDevice, st));
    int e = ccd_ssim_launch(reinterpret_cast<const SsimJobDev *>(A.dv + off_jobs), n_jobs, max_tiles, g, st);
    if (e != 0) return fail(CCD_ERR_CUDA, "MS-SSIM launch failed: %s", cudaGetErrorString((cudaError_t)e));
    if (int rc = download(A, off_bad, st, "MS-SSIM")) return rc;
    const double *part = reinterpret_cast<const double *>(A.h + off_part);
    for (int i = 0; i < n_jobs; i++) {
        for (int j = 0; j < S; j++) {
            const double *p = part + 2 * part_at[(size_t)i * S + j];  // the planes' tiles in order
            for (int c = 0; c < 3; c++) {
                const size_t t = (size_t)tiles(i, c, j);
                const double n_pos = (double)(side(i, c, j, false) - CCD_SSIM_HALO) * (side(i, c, j, true) - CCD_SSIM_HALO);
                jobs[i].cs[c][j] = ordered_sum(p, t, 2) / n_pos;
                jobs[i].ssim[c][j] = ordered_sum(p + 1, t, 2) / n_pos;
                p += 2 * t;
            }
        }
    }
    return report(jobs, n_jobs, reinterpret_cast<const unsigned long long *>(A.h + off_bad), [&](int i) { return off_grid_error(jobs[i], i); });
}

int ccd_frame_ssim(CcdContext *ctx, CcdSsimJob *jobs, int n_jobs, void *cuda_stream) {
    return job_call(ctx, jobs, n_jobs, cuda_stream, [&](cudaStream_t st) -> int { return frame_ssim_body(ctx, jobs, n_jobs, st); });
}

int ccd_finish_frame(CcdContext *ctx, const float *d_in, int h, int w, int bitdepth, int data_type, float *d_out_a,
                     float *d_out_b, float *d_out_c, void *cuda_stream) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        if (!d_in || !d_out_a || h < 1 || w < 1 || bitdepth < 8 || bitdepth > 16 || data_type < 0 || data_type > 2)
            return fail(CCD_ERR_ARG, "bad argument");
        if (data_type == 1 && (!d_out_b || !d_out_c)) return fail(CCD_ERR_ARG, "yuv420 needs u and v outputs");
        if (ccd_finish(d_in, h, w, bitdepth, data_type, d_out_a, d_out_b, d_out_c, st))
            return fail(CCD_ERR_CUDA, "finish_frame launch failed");
        return CCD_OK;
    });
}

namespace {
// The launch arguments of a P/B frame, with every check of the reconstruction and of the statistics (outputs aside).
int inter_launch_args(const CcdInterFrame *f, InterLaunch &L) {
    if (!f || !f->d_residue || !f->d_motion || !f->ref0[0] || !f->ref0[1] || !f->ref0[2] || f->h < 1 || f->w < 1)
        return fail(CCD_ERR_ARG, "bad argument");
    const int is_b = f->is_b;
    if (f->bitdepth < 0 || f->bitdepth > 16) return fail(CCD_ERR_ARG, "bad bitdepth %d", f->bitdepth);
    if (f->frame_data_type < 0 || f->frame_data_type > 3) return fail(CCD_ERR_ARG, "bad frame_data_type %d", f->frame_data_type);
    if (f->bitdepth == 0 && f->frame_data_type == 1) return fail(CCD_ERR_ARG, "the pre-rounding frame takes 4:4:4 references");
    if (is_b && (!f->ref1[0] || !f->ref1[1] || !f->ref1[2])) return fail(CCD_ERR_ARG, "B frame without a second reference");
    // decode.py:171-189 reads residue channels 0..3 (P) / 0..4 (B) and motion channels 0..1 (P) / 0..3 (B)
    if (f->n_res_ch != (is_b ? 5 : 4))
        return fail(CCD_ERR_ARG, "%s-frame residue has %d channels, expected %d", is_b ? "B" : "P", f->n_res_ch, is_b ? 5 : 4);
    if (f->n_mot_ch != (is_b ? 4 : 2))
        return fail(CCD_ERR_ARG, "%s-frame motion has %d channels, expected %d", is_b ? "B" : "P", f->n_mot_ch, is_b ? 4 : 2);
    if (f->frame_data_type == 1 && ((f->h | f->w) & 1)) return fail(CCD_ERR_ARG, "4:2:0 needs even frame sizes, got %dx%d", f->h, f->w);
    if (f->warp_filter_size < 2 || (f->warp_filter_size & 1)) return fail(CCD_ERR_ARG, "bad warp filter size %d", f->warp_filter_size);
    L = InterLaunch{};
    L.residue = f->d_residue;
    L.motion = f->d_motion;
    for (int c = 0; c < 3; c++) {
        L.ref0[c] = f->ref0[c];
        L.ref1[c] = is_b ? f->ref1[c] : nullptr;
    }
    L.ref_cs = L.out_420 = (f->frame_data_type == 1);
    L.h = f->h;
    L.w = f->w;
    L.is_b = is_b;
    for (int i = 0; i < 4; i++) L.gf[i] = (i < 2 || is_b) ? f->global_flow[i] : 0;
    L.filter_size = f->warp_filter_size;
    L.M = f->bitdepth ? (float)((1 << f->bitdepth) - 1) : 0.0f;
    return CCD_OK;
}

// status of a P/B kernel launch (ccd_inter_launch, ccd_inter_stats_launch)
int inter_launched(int rc, int filter_size) {
    if (rc == -1)
        return fail(CCD_ERR_UNSUPPORTED, "warp filter size %d is not supported (2, 4: frames of at least 2x2; 6 .. 14)", filter_size);
    if (rc) return fail(CCD_ERR_CUDA, "P/B kernel launch failed: %s", cudaGetErrorString((cudaError_t)rc));
    return CCD_OK;
}
}  // namespace

int ccd_reconstruct_frame(CcdContext *ctx, const CcdInterFrame *frame, float *const out_planes[3], void *cuda_stream) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        InterLaunch L;
        if (int rc = inter_launch_args(frame, L)) return rc;
        if (!out_planes || !out_planes[0] || !out_planes[1] || !out_planes[2]) return fail(CCD_ERR_ARG, "bad argument");
        for (int c = 0; c < 3; c++) L.out[c] = out_planes[c];
        return inter_launched(ccd_inter_launch(L, st), L.filter_size);
    });
}

int ccd_inter_stats(CcdContext *ctx, const CcdInterFrame *frame, CcdInterStats *stats, void *cuda_stream) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        InterLaunch L;
        if (int rc = inter_launch_args(frame, L)) return rc;
        if (!stats) return fail(CCD_ERR_ARG, "bad argument");
        if (frame->bitdepth < 1) return fail(CCD_ERR_ARG, "bad bitdepth %d", frame->bitdepth);
        const int layout = stats->src_layout;
        if (layout < 0 || layout > 1 || (layout == 1 && frame->frame_data_type == 1))
            return fail(CCD_ERR_ARG, "bad source layout %d for frame_data_type %d", layout, frame->frame_data_type);
        const int64_t n_ctas = ccd_inter_stats_ctas(L.h, L.w);
        Arena A;  // results only: the partials, which need no initial value (nothing is uploaded)
        const size_t off_part = A.take(sizeof(double) * 4 * (size_t)n_ctas);
        if (int rc = stage(ctx, A)) return rc;
        InterStatsOut o{};
        o.src = stats->d_src;
        o.src_hwc = layout;
        o.src_wide = frame->bitdepth > 8;
        o.src_M = L.M;
        o.alpha = stats->d_alpha;
        o.beta = stats->d_beta;
        o.pred = stats->d_pred;
        o.part = reinterpret_cast<double *>(A.dv + off_part);
        if (int rc = inter_launched(ccd_inter_stats_launch(L, o, st), L.filter_size)) return rc;
        if (int rc = download(A, off_part, st, "inter_stats")) return rc;
        const double *part = reinterpret_cast<const double *>(A.h + off_part);
        for (int k = 0; k < 4; k++) stats->sums[k] = ordered_sum(part + k, (size_t)n_ctas, 4);  // CTAs in order
        return CCD_OK;
    });
}

int ccd_pack_frame(CcdContext *ctx, const float *const planes[3], int h, int w, int chroma_shift, int bitdepth,
                   int sample_bytes, int interleaved, void *d_out, void *cuda_stream) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        if (!planes || !planes[0] || !planes[1] || !planes[2] || !d_out || h < 1 || w < 1) return fail(CCD_ERR_ARG, "bad argument");
        if (bitdepth < 1 || bitdepth > 16 || (sample_bytes != 1 && sample_bytes != 2) || (sample_bytes == 1 && bitdepth > 8))
            return fail(CCD_ERR_ARG, "bitdepth %d does not fit %d-byte samples", bitdepth, sample_bytes);
        if (chroma_shift < 0 || chroma_shift > 1 || (interleaved && chroma_shift)) return fail(CCD_ERR_ARG, "bad layout");
        if (ccd_pack(planes, h, w, chroma_shift, bitdepth, sample_bytes, interleaved, d_out, st))
            return fail(CCD_ERR_CUDA, "pack_frame launch failed");
        return CCD_OK;
    });
}

int ccd_pack_samples(CcdContext *ctx, const float *d_samples, size_t n, int bitdepth, int sample_bytes, void *d_out,
                     void *cuda_stream) {
    return guarded(ctx, cuda_stream, [&](cudaStream_t st) -> int {
        if (!d_samples || !d_out || n == 0) return fail(CCD_ERR_ARG, "bad argument");
        if (bitdepth < 1 || bitdepth > 16 || (sample_bytes != 1 && sample_bytes != 2) || (sample_bytes == 1 && bitdepth > 8))
            return fail(CCD_ERR_ARG, "bitdepth %d does not fit %d-byte samples", bitdepth, sample_bytes);
        if (ccd_pack_flat(d_samples, n, bitdepth, sample_bytes, d_out, st)) return fail(CCD_ERR_CUDA, "pack_samples launch failed");
        return CCD_OK;
    });
}

int ccd_debug_laplace_domain(CcdContext *ctx, int sc_lo, int sc_hi, uint32_t *out_lo, uint32_t *out_hi) {
    return guarded(ctx, nullptr, [&](cudaStream_t st) -> int {
        if (sc_lo < 0 || sc_hi > CCD_N_SCALE || sc_lo >= sc_hi || !out_lo || !out_hi) return fail(CCD_ERR_ARG, "bad argument");
        const size_t n = (size_t)(sc_hi - sc_lo) * 32641;
        if (int rc = ensure_dev(ctx->scratch, n * 8)) return rc;
        uint32_t *lo = reinterpret_cast<uint32_t *>(ctx->scratch.p), *hi = lo + n;
        if (ccd_laplace_domain(ctx->d_scale, sc_lo, sc_hi, lo, hi, st)) return fail(CCD_ERR_CUDA, "launch failed");
        CUDA_TRY(cudaMemcpy(out_lo, lo, n * 4, cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(out_hi, hi, n * 4, cudaMemcpyDeviceToHost));
        return CCD_OK;
    });
}

uint64_t ccd_debug_launch_count(void) { return g_ccd_launches; }

int ccd_debug_entropy_plan(const CcdCoolChicDesc *desc, const int64_t *nn_ints, int64_t out[3]) {
    if (!desc || !nn_ints || !out) return fail(CCD_ERR_ARG, "null pointer");
    PreparedJob P;
    P.d = desc;
    if (int rc = prepare_job(P, nn_ints)) return rc;
    out[0] = P.es.ring;
    out[1] = P.es.rows;
    out[2] = (int64_t)P.smem;
    return entropy_smem_ok(P.smem);
}

int ccd_debug_set_producer_mask(CcdContext *ctx, uint32_t mask) {
    if (!ctx || (mask & 0x3fffu) == 0) return fail(CCD_ERR_ARG, "bad producer mask");
    ctx->prod_mask = mask & 0x3fffu;
    return CCD_OK;
}

int ccd_debug_last_status(const CcdContext *ctx, int32_t st[16]) {
    if (!ctx || !st) return fail(CCD_ERR_ARG, "null pointer");
    memcpy(st, ctx->last_status, 64);
    return CCD_OK;
}

int ccd_last_timing(const CcdContext *ctx, float ms[4]) {
    if (!ctx || !ms) return fail(CCD_ERR_ARG, "null pointer");
    memcpy(ms, ctx->last_ms, sizeof(float) * 4);
    ms[3] = (float)ctx->last_upload_bytes;
    return CCD_OK;
}

}  // extern "C"
