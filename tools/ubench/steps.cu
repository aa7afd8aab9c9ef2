// Micro-benchmark: candidate per-symbol steps of the range-coder warp, one warp, with / without "producer-like"
// noise warps on the same SM.  Every symbol is the mode and no renormalisation occurs (hot entry (0, 0, 2^24, 2^24):
// R keeps its magnitude), so the loop-carried chain is exactly the arithmetic under test.
//   usage: ./steps            (prints cycles / symbol for every variant, noise 0 and 11)
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t lds(uint32_t a){uint32_t v; asm volatile("ld.volatile.shared.u32 %0,[%1];":"=r"(v):"r"(a):"memory"); return v;}
__device__ __forceinline__ void sts(uint32_t a, uint32_t v){asm volatile("st.volatile.shared.u32 [%0],%1;"::"r"(a),"r"(v):"memory");}
__device__ __forceinline__ uint4 lds4(uint32_t a){uint4 v; asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3},[%4];":"=r"(v.x),"=r"(v.y),"=r"(v.z),"=r"(v.w):"r"(a):"memory"); return v;}

// V0: mode only, flag accumulated (tier 1 of a speculative design): h.y = left(M), h.z - h.y = p(M)
__device__ __forceinline__ uint32_t step_mode(uint64_t &D, uint64_t &R, uint4 h) {
    const uint64_t s = R >> 24;
    const uint64_t lo = s * h.y, rn = s * (h.z - h.y);
    const uint64_t dn = D - lo;
    const uint32_t bad = (uint32_t)(dn >> 32) >= (uint32_t)(rn >> 32);
    D = dn; R = rn;
    return bad;
}
// V2: three candidates, 64-bit compares then two-level selects (no renormalisation)
__device__ __forceinline__ uint32_t step_cmp(uint64_t &D, uint64_t &R, uint4 h, uint32_t &t) {
    const uint64_t s = R >> 24;
    const uint64_t P0 = s * h.x, P1 = s * h.y, P2 = s * h.z, P3 = s * h.w;
    const bool c1 = D >= P1, c2 = D >= P2;
    const uint32_t far = (uint32_t)(D < P0) | (uint32_t)(D >= P3);
    const uint64_t nlo = c2 ? P2 : (c1 ? P1 : P0);
    const uint64_t nhi = c2 ? P3 : (c1 ? P2 : P1);
    D = D - nlo; R = nhi - nlo;
    t = c2 ? 15u : (c1 ? 14u : 13u);
    return far;
}
// V3: three candidates, differences E_i = D - P_i (borrow = compare), selects among the differences; R from products of p
__device__ __forceinline__ uint32_t step_diff(uint64_t &D, uint64_t &R, uint4 h, uint32_t &t) {
    const uint64_t s = R >> 24;
    const uint64_t P0 = s * h.x, P1 = s * h.y, P2 = s * h.z, P3 = s * h.w;
    const uint64_t Q0 = P1 - P0, Q1 = P2 - P1, Q2 = P3 - P2;
    const uint64_t E0 = D - P0, E1 = D - P1, E2 = D - P2;
    const bool c1 = D >= P1, c2 = D >= P2;
    const uint32_t far = (uint32_t)(D < P0) | (uint32_t)(D >= P3);
    D = c2 ? E2 : (c1 ? E1 : E0);
    R = c2 ? Q2 : (c1 ? Q1 : Q0);
    t = c2 ? 15u : (c1 ? 14u : 13u);
    return far;
}
// V4: V2 + renormalisation by selects (word from a register)
__device__ __forceinline__ uint32_t step_cmp_rn(uint64_t &D, uint64_t &R, uint4 h, uint32_t &t, uint32_t w0, uint32_t &wpos) {
    const uint64_t s = R >> 24;
    const uint64_t P0 = s * h.x, P1 = s * h.y, P2 = s * h.z, P3 = s * h.w;
    const bool c1 = D >= P1, c2 = D >= P2;
    const uint32_t far = (uint32_t)(D < P0) | (uint32_t)(D >= P3);
    const uint64_t nlo = c2 ? P2 : (c1 ? P1 : P0);
    const uint64_t nhi = c2 ? P3 : (c1 ? P2 : P1);
    const uint64_t Dn = D - nlo, Rn = nhi - nlo;
    const bool rn = (uint32_t)(Rn >> 32) == 0u;
    D = rn ? ((Dn << 32) | w0) : Dn;
    R = rn ? (Rn << 32) : Rn;
    wpos += rn ? 1u : 0u;
    t = c2 ? 15u : (c1 ? 14u : 13u);
    return far;
}
// V6: V0 with a taken branch per block of K steps (in k below)
// V5: mode first with ONE select level: R' = mode ? Q1 : Qx where Qx = (D < P1) ? Q0 : Q2 is formed off the mode chain
__device__ __forceinline__ uint32_t step_mode_first(uint64_t &D, uint64_t &R, uint4 h, uint32_t &t) {
    const uint64_t s = R >> 24;
    const uint64_t P0 = s * h.x, P1 = s * h.y, P2 = s * h.z, P3 = s * h.w;
    const uint64_t E1 = D - P1;                     // wraps when D < P1
    const uint64_t Q1 = P2 - P1;
    const bool below = D < P1;
    const bool is_m = E1 < Q1;                      // P1 <= D < P2 (wrapping compare)
    const uint64_t Ex = below ? D - P0 : D - P2;
    const uint64_t Qx = below ? P1 - P0 : P3 - P2;
    const uint32_t far = is_m ? 0u : (uint32_t)(Ex >= Qx);
    D = is_m ? E1 : Ex;
    R = is_m ? Q1 : Qx;
    t = is_m ? 14u : (below ? 13u : 15u);
    return far;
}

template <int VAR, int K>
__global__ void k(long long *out, int n, int noise) {
    extern __shared__ __align__(16) unsigned char smraw[];
    uint32_t base = (uint32_t)__cvta_generic_to_shared(smraw);
    asm volatile("" : "+r"(base));
    const uint32_t RING = 256, hot = base + 64, ctrl = base, mask = RING - 1;
    for (int i = threadIdx.x; i < 512; i += blockDim.x) ((uint4 *)(smraw + 64))[i] = make_uint4(0u, 0u, 16777216u, 16777216u);
    if (threadIdx.x == 0) { ((volatile uint32_t *)smraw)[0] = 0; ((volatile uint32_t *)smraw)[1] = 0x7fffffff; }
    __syncthreads();
    const int warp = threadIdx.x >> 5;
    if (warp != 15) {
        if (warp >= noise || (warp & 3) == 3) return;  // like the product: the coder's scheduler partition stays empty
        uint32_t acc = threadIdx.x;
        while ((int)lds(ctrl) >= 0) { for (int q = 0; q < 16; q++) acc = acc * 1664525u + lds(hot + ((acc >> 8) & 0xff0)); }
        if (acc == 0x12345) out[5] = acc;
        return;
    }
    uint64_t D = 0x0000123456789abcull, R = 0x00dcba9876543210ull;
    uint32_t j = 0, bad_all = 0, tsum = 0, wpos = 0;
    const uint32_t end = (uint32_t)n;
    uint32_t o = hot + (j & mask) * 16u;
    uint4 a[K], b[K];
#pragma unroll
    for (int i = 0; i < K; i++) a[i] = lds4(o + 16u * i);
    uint32_t badp = 0;
    const long long t0 = clock64();
    while (j < end) {
        o = hot + ((j + K) & mask) * 16u;
#pragma unroll
        for (int i = 0; i < K; i++) b[i] = lds4(o + 16u * i);
        uint32_t bad = 0, tt = 0;
#pragma unroll
        for (int i = 0; i < K; i++) {
            uint32_t t = 14u;
            if (VAR == 0 || VAR == 1 || VAR == 6) bad |= step_mode(D, R, a[i]);
            else if (VAR == 2) bad |= step_cmp(D, R, a[i], t);
            else if (VAR == 3) bad |= step_diff(D, R, a[i], t);
            else if (VAR == 4) bad |= step_cmp_rn(D, R, a[i], t, 0x12345678u, wpos);
            else if (VAR == 5) bad |= step_mode_first(D, R, a[i], t);
            tt |= t << (8 * i);
        }
        if (VAR == 1) { if (bad) { bad_all++; D ^= 1; } }          // fresh predicate
        else { if (badp) { bad_all++; D ^= 1; } }                 // verified one group late
        if (VAR == 6) {
            // a block on fresh data that is never entered, too long to predicate: ptxas places it in line, so the branch
            // around it is taken once per block; V6 - V0 = the cost of one taken branch to this warp
            if ((uint32_t)(D >> 8) == 0x12345u) {
                uint32_t x = (uint32_t)R;
#pragma unroll
                for (int q = 0; q < 24; q++) x = x * 1664525u + (uint32_t)(D >> q);
                bad_all += x;
            }
        }
        badp = bad;
        tsum += tt;
        sts(ctrl + 8, j);
        j += K;
#pragma unroll
        for (int i = 0; i < K; i++) a[i] = b[i];
    }
    const long long t1 = clock64();
    if ((threadIdx.x & 31) == 0) { out[0] = t1 - t0; out[1] = (long long)(D ^ R) + bad_all + tsum + wpos; }
    sts(ctrl, 0x80000000u);
}

template <int VAR, int K> void run(const char *name, long long *d_out) {
    const int n = 1 << 20;
    cudaFuncSetAttribute(k<VAR, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 + 512 * 16);
    for (int noise : {0, 14}) {
        long long h[2] = {0, 0};
        for (int rep = 0; rep < 2; rep++) {
            k<VAR, K><<<1, 512, 64 + 512 * 16>>>(d_out, n, noise);
            cudaDeviceSynchronize();
            cudaMemcpy(h, d_out, 16, cudaMemcpyDeviceToHost);
        }
        printf("%-34s K=%d noise=%2d : %7.1f cycles / symbol   (err %s)\n", name, K, noise, (double)h[0] / n, cudaGetErrorString(cudaGetLastError()));
    }
}

int main() {
    long long *d_out;
    cudaMalloc(&d_out, 64);
    run<0, 4>("mode only, lagged check", d_out);
    run<1, 4>("mode only, fresh check", d_out);
    run<0, 2>("mode only, lagged check", d_out);
    run<0, 8>("mode only, lagged check", d_out);
    run<6, 4>("mode only, taken branch per block", d_out);
    run<6, 2>("mode only, taken branch per block", d_out);
    run<2, 4>("3 cand, compare + 2-level select", d_out);
    run<3, 4>("3 cand, differences", d_out);
    run<4, 4>("3 cand, compare + renorm selects", d_out);
    run<5, 4>("3 cand, mode first", d_out);
    run<5, 2>("3 cand, mode first", d_out);
    return 0;
}
