// Causal attention of the event-level stack (head_dim 64) on the Hopper tensor cores, forward and backward
// (hf sdpa_attention.py:92-101 called from modeling_llama.py:251-289 with is_causal=True, scale = d^-1/2).
// One warpgroup per CTA owns a 64-row tile; Q / K / V / dO tiles of 64 x 64 bf16 are staged by TMA (3-D tensor maps
// {columns, rows, batch}: rows past the end of a sequence are zero-filled) into 128B-swizzled shared memory, double
// buffered through mbarriers.  Every product is wgmma m64n64k16 with fp32 accumulators in registers; the second product
// of each pair (P.V, dS.K, ...) takes its A operand straight from the first one's accumulators (the fragment layouts
// coincide), so P and dS never touch shared memory.
//   fwd : CTA = 64 query rows x (batch, head); online softmax in fp32, P rounded to bf16 before P.V, output rounded to
//         bf16, LSE saved for the backward pass
//   dkv : CTA = 64 keys x (batch, head), loops over query tiles: dV += P^T dO, dK += dS^T Q   (no atomics)
//   dq  : CTA = 64 query rows x (batch, head), loops over key tiles: dQ += dS K                (no atomics)
// The RoPE backward can be fused into the dK / dQ stores (gradient w.r.t. the pre-rotation projections).
// Same semantics as the mma.sync kernels of attn_flash.cu, which the tests use as the second implementation.
#include "hopper.cuh"

namespace {
using namespace hopper;

constexpr int D = 64;
constexpr int T = 64;                  // rows per tile (queries or keys)
constexpr int NT = 128;                // one warpgroup
constexpr int TILE_BYTES = T * D * 2;  // 8 KB
constexpr float LOG2E = 1.4426950408889634f;

struct Strides {
    long long b, r, h;
};

struct Params {
    int n_heads, Sq, Sk, off;          // off = Sk - Sq: query row q sees keys <= q + off
    float scale;
};

// K-major tile [64 rows][64 d] as an operand whose reduction dimension is d: k-step kk = 16 d = 32 bytes
__device__ __forceinline__ uint64_t desc_kmaj(uint32_t base, int kk) { return make_smem_desc(base + kk * 32, 16, 1024); }
// the same tile as an operand whose reduction dimension is its rows (N = d): k-step kk = 16 rows = 2 KB
__device__ __forceinline__ uint64_t desc_mnmaj(uint32_t base, int kk) { return make_smem_desc(base + kk * 2048, 8192, 1024); }

// acc(64 x 64) = A(64 x 64 d) . B(64 x 64 d)^T, both K-major tiles in shared memory
__device__ __forceinline__ void mma_tt(float* acc, uint32_t a, uint32_t b) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; kk++) wgmma_m64n64k16<0, 0>(acc, desc_kmaj(a, kk), desc_kmaj(b, kk), kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
}
// acc(64 x 64 d) += P(64 x 64, bf16 fragments) . B(64 rows x 64 d)
__device__ __forceinline__ void mma_pv(float* acc, const uint32_t (*pa)[4], uint32_t b) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; kk++) wgmma_m64n64k16_rs<1>(acc, pa[kk], desc_mnmaj(b, kk), 1u);
    wgmma_commit();
    wgmma_wait<0>();
}
// accumulator fragment (64 x 64 fp32) -> A fragments of four k16 chunks (bf16)
__device__ __forceinline__ void to_afrag(const float* s, uint32_t (*pa)[4]) {
#pragma unroll
    for (int kk = 0; kk < 4; kk++)
#pragma unroll
        for (int i = 0; i < 4; i++) pa[kk][i] = pack2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
}

// RoPE backward on a 64-column accumulator row half h: (d, d + 32) pairs are groups (nb, nb + 4) of the same thread
__device__ __forceinline__ void rope_bwd(float* acc, int h, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                         int pos, int cq) {
#pragma unroll
    for (int nb = 0; nb < 4; nb++) {
        const float2 c = __bfloat1622float2(*reinterpret_cast<const bf162*>(cos_t + (size_t)pos * 32 + nb * 8 + cq));
        const float2 sn = __bfloat1622float2(*reinterpret_cast<const bf162*>(sin_t + (size_t)pos * 32 + nb * 8 + cq));
        float* a = acc + 4 * nb + 2 * h;
        float* b = acc + 4 * (nb + 4) + 2 * h;
        const float a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
        a[0] = a0 * c.x + b0 * sn.x;
        a[1] = a1 * c.y + b1 * sn.y;
        b[0] = b0 * c.x - a0 * sn.x;
        b[1] = b1 * c.y - a1 * sn.y;
    }
}

__device__ __forceinline__ uint8_t* smem_base() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
}

// ------------------------------------------------------------------------------------------------ forward
// smem: Q | K[2] | V[2] | barriers
__global__ void __launch_bounds__(NT)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, bf16* __restrict__ o, float* __restrict__ lse, Strides so,
                      const Params p) {
    uint8_t* sm = smem_base();
    uint8_t* sQ = sm;
    uint8_t* sK = sm + TILE_BYTES;
    uint8_t* sV = sK + 2 * TILE_BYTES;
    uint64_t* bar = reinterpret_cast<uint64_t*>(sV + 2 * TILE_BYTES);     // [0]: Q, [1 + s]: K/V stage s
    const int bh = blockIdx.x, b = bh / p.n_heads, h = bh % p.n_heads;
    const int q_blk = gridDim.y - 1 - blockIdx.y;                          // longest rows first
    const int q0 = q_blk * T;
    const int last_key = min(q0 + T - 1 + p.off, p.Sk - 1);
    const int nk = last_key / T + 1;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
    if (tid == 0) {
        for (int i = 0; i < 3; i++) mbar_init(&bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&bar[0], TILE_BYTES);
        tma_load_3d(sQ, &tmQ, &bar[0], h * D, q0, b);
        mbar_expect_tx(&bar[1], 2 * TILE_BYTES);
        tma_load_3d(sK, &tmK, &bar[1], h * D, 0, b);
        tma_load_3d(sV, &tmV, &bar[1], h * D, 0, b);
    }
    __syncthreads();
    float oacc[32], s[32];
#pragma unroll
    for (int i = 0; i < 32; i++) oacc[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const float sl2 = p.scale * LOG2E;
    const int r0 = warp * 16 + (lane >> 2);
    mbar_wait(&bar[0], 0);
    for (int j = 0; j < nk; j++) {
        const int st = j & 1;
        if (tid == 0 && j + 1 < nk) {           // stage st ^ 1 was released by the barrier that ended iteration j - 1
            mbar_expect_tx(&bar[1 + (st ^ 1)], 2 * TILE_BYTES);
            tma_load_3d(sK + (st ^ 1) * TILE_BYTES, &tmK, &bar[1 + (st ^ 1)], h * D, (j + 1) * T, b);
            tma_load_3d(sV + (st ^ 1) * TILE_BYTES, &tmV, &bar[1 + (st ^ 1)], h * D, (j + 1) * T, b);
        }
        mbar_wait(&bar[1 + st], (j >> 1) & 1);
        mma_tt(s, smem_u32(sQ), smem_u32(sK + st * TILE_BYTES));
        const int k0 = j * T;
        const bool edge = k0 + T - 1 > q0 + p.off || k0 + T > p.Sk;
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const int q = q0 + r0 + 8 * hh;
            float mx = -INFINITY;
#pragma unroll
            for (int g = 0; g < 8; g++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    float& x = s[4 * g + 2 * hh + e];
                    const int key = k0 + 8 * g + cq + e;
                    x = (edge && (key > q + p.off || key >= p.Sk)) ? -INFINITY : x * sl2;
                    mx = fmaxf(mx, x);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float mn = fmaxf(m[hh], mx);
            const float alpha = exp2f(m[hh] - mn);
            m[hh] = mn;
            float sum = 0.f;
#pragma unroll
            for (int g = 0; g < 8; g++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    float& x = s[4 * g + 2 * hh + e];
                    x = exp2f(x - mn);
                    sum += x;
                    oacc[4 * g + 2 * hh + e] *= alpha;
                }
            l[hh] = l[hh] * alpha + sum;
        }
        uint32_t pa[4][4];
        to_afrag(s, pa);
        mma_pv(oacc, pa, smem_u32(sV + st * TILE_BYTES));
        __syncthreads();
    }
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        float t = l[hh];
        t += __shfl_xor_sync(0xffffffffu, t, 1);
        t += __shfl_xor_sync(0xffffffffu, t, 2);
        const int q = q0 + r0 + 8 * hh;
        if (q < p.Sq) {
            const float inv = 1.f / t;
            bf16* dst = o + b * so.b + (long long)q * so.r + h * so.h + cq;
#pragma unroll
            for (int g = 0; g < 8; g++)
                *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack2(oacc[4 * g + 2 * hh] * inv, oacc[4 * g + 2 * hh + 1] * inv);
            if (lse && (lane & 3) == 0) lse[((long long)b * p.n_heads + h) * p.Sq + q] = (m[hh] + log2f(t)) / LOG2E;
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward dK, dV
// smem: K | V | Q[2] | dO[2] | lse[2][64] | delta[2][64] | barriers
__global__ void __launch_bounds__(NT)
attn_bwd_dkv_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                          const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dk,
                          bf16* __restrict__ dv, Strides sdk, Strides sdv, const Params p, const bf16* __restrict__ rope_cos,
                          const bf16* __restrict__ rope_sin) {
    uint8_t* sm = smem_base();
    uint8_t* sK = sm;
    uint8_t* sV = sm + TILE_BYTES;
    uint8_t* sQ = sV + TILE_BYTES;
    uint8_t* sdO = sQ + 2 * TILE_BYTES;
    float* s_lse = reinterpret_cast<float*>(sdO + 2 * TILE_BYTES);   // [2][64], already in log2 units
    float* s_del = s_lse + 2 * T;                                   // [2][64]
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_del + 2 * T);     // [0]: K/V, [1 + s]: Q/dO stage s
    const int bh = blockIdx.x, b = bh / p.n_heads, h = bh % p.n_heads;
    const int k0 = blockIdx.y * T;
    const int q_first = max(0, k0 - p.off) / T;
    const int q_end = (p.Sq + T - 1) / T;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
    const float* lse_g = lse + (long long)bh * p.Sq;
    const float* del_g = delta + (long long)bh * p.Sq;
    if (tid == 0) {
        for (int i = 0; i < 3; i++) mbar_init(&bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&bar[0], 2 * TILE_BYTES);
        tma_load_3d(sK, &tmK, &bar[0], h * D, k0, b);
        tma_load_3d(sV, &tmV, &bar[0], h * D, k0, b);
        if (q_first < q_end) {
            mbar_expect_tx(&bar[1], 2 * TILE_BYTES);
            tma_load_3d(sQ, &tmQ, &bar[1], h * D, q_first * T, b);
            tma_load_3d(sdO, &tmdO, &bar[1], h * D, q_first * T, b);
        }
    }
    float dkacc[32], dvacc[32], s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; i++) dkacc[i] = dvacc[i] = 0.f;
    const float sl2 = p.scale * LOG2E;
    const int r0 = warp * 16 + (lane >> 2);
    __syncthreads();
    mbar_wait(&bar[0], 0);
    for (int it = 0, qb = q_first; qb < q_end; it++, qb++) {
        const int st = it & 1;
        const int q0 = qb * T;
        if (tid == 0 && qb + 1 < q_end) {
            mbar_expect_tx(&bar[1 + (st ^ 1)], 2 * TILE_BYTES);
            tma_load_3d(sQ + (st ^ 1) * TILE_BYTES, &tmQ, &bar[1 + (st ^ 1)], h * D, q0 + T, b);
            tma_load_3d(sdO + (st ^ 1) * TILE_BYTES, &tmdO, &bar[1 + (st ^ 1)], h * D, q0 + T, b);
        }
        if (tid < T) s_lse[st * T + tid] = q0 + tid < p.Sq ? lse_g[q0 + tid] * LOG2E : 0.f;
        else s_del[st * T + tid - T] = q0 + tid - T < p.Sq ? del_g[q0 + tid - T] : 0.f;
        __syncthreads();
        mbar_wait(&bar[1 + st], (it >> 1) & 1);
        const uint32_t aQ = smem_u32(sQ + st * TILE_BYTES), adO = smem_u32(sdO + st * TILE_BYTES);
        mma_tt(s, smem_u32(sK), aQ);             // S^T = K Q^T   (rows = keys, columns = queries)
        mma_tt(dp, smem_u32(sV), adO);           // dP^T = V dO^T
        const bool edge = k0 + T - 1 > q0 + p.off || q0 + T > p.Sq;
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const int key = k0 + r0 + 8 * hh;
#pragma unroll
            for (int g = 0; g < 8; g++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int i = 4 * g + 2 * hh + e, qc = 8 * g + cq + e, q = q0 + qc;
                    const bool dead = edge && (key > q + p.off || q >= p.Sq);
                    const float pr = dead ? 0.f : exp2f(s[i] * sl2 - s_lse[st * T + qc]);
                    s[i] = pr;
                    dp[i] = pr * (dp[i] - s_del[st * T + qc]);
                }
        }
        uint32_t pa[4][4];
        to_afrag(s, pa);
        mma_pv(dvacc, pa, adO);                   // dV += P^T dO
        to_afrag(dp, pa);
        mma_pv(dkacc, pa, aQ);                    // dK += dS^T Q
        __syncthreads();
    }
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        const int key = k0 + r0 + 8 * hh;
        if (key < p.Sk) {
            if (rope_cos) rope_bwd(dkacc, hh, rope_cos, rope_sin, key, cq);   // linear: commutes with the scale below
            bf16* dkg = dk + b * sdk.b + (long long)key * sdk.r + h * sdk.h + cq;
            bf16* dvg = dv + b * sdv.b + (long long)key * sdv.r + h * sdv.h + cq;
#pragma unroll
            for (int g = 0; g < 8; g++) {
                *reinterpret_cast<uint32_t*>(dkg + 8 * g) = pack2(dkacc[4 * g + 2 * hh] * p.scale, dkacc[4 * g + 2 * hh + 1] * p.scale);
                *reinterpret_cast<uint32_t*>(dvg + 8 * g) = pack2(dvacc[4 * g + 2 * hh], dvacc[4 * g + 2 * hh + 1]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward dQ
// smem: Q | dO | K[2] | V[2] | barriers
__global__ void __launch_bounds__(NT)
attn_bwd_dq_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                         const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                         const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dq, Strides sdq,
                         const Params p, const bf16* __restrict__ rope_cos, const bf16* __restrict__ rope_sin) {
    uint8_t* sm = smem_base();
    uint8_t* sQ = sm;
    uint8_t* sdO = sm + TILE_BYTES;
    uint8_t* sK = sdO + TILE_BYTES;
    uint8_t* sV = sK + 2 * TILE_BYTES;
    uint64_t* bar = reinterpret_cast<uint64_t*>(sV + 2 * TILE_BYTES);     // [0]: Q/dO, [1 + s]: K/V stage s
    const int bh = blockIdx.x, b = bh / p.n_heads, h = bh % p.n_heads;
    const int q0 = (gridDim.y - 1 - blockIdx.y) * T;
    const int nk = min(q0 + T - 1 + p.off, p.Sk - 1) / T + 1;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
    if (tid == 0) {
        for (int i = 0; i < 3; i++) mbar_init(&bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&bar[0], 2 * TILE_BYTES);
        tma_load_3d(sQ, &tmQ, &bar[0], h * D, q0, b);
        tma_load_3d(sdO, &tmdO, &bar[0], h * D, q0, b);
        mbar_expect_tx(&bar[1], 2 * TILE_BYTES);
        tma_load_3d(sK, &tmK, &bar[1], h * D, 0, b);
        tma_load_3d(sV, &tmV, &bar[1], h * D, 0, b);
    }
    const int r0 = warp * 16 + (lane >> 2);
    float lse_r[2], del_r[2];
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        const int q = q0 + r0 + 8 * hh;
        lse_r[hh] = q < p.Sq ? lse[(long long)bh * p.Sq + q] * LOG2E : 0.f;
        del_r[hh] = q < p.Sq ? delta[(long long)bh * p.Sq + q] : 0.f;
    }
    float dqacc[32], s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; i++) dqacc[i] = 0.f;
    const float sl2 = p.scale * LOG2E;
    __syncthreads();
    mbar_wait(&bar[0], 0);
    for (int j = 0; j < nk; j++) {
        const int st = j & 1;
        if (tid == 0 && j + 1 < nk) {
            mbar_expect_tx(&bar[1 + (st ^ 1)], 2 * TILE_BYTES);
            tma_load_3d(sK + (st ^ 1) * TILE_BYTES, &tmK, &bar[1 + (st ^ 1)], h * D, (j + 1) * T, b);
            tma_load_3d(sV + (st ^ 1) * TILE_BYTES, &tmV, &bar[1 + (st ^ 1)], h * D, (j + 1) * T, b);
        }
        mbar_wait(&bar[1 + st], (j >> 1) & 1);
        const uint32_t aK = smem_u32(sK + st * TILE_BYTES);
        mma_tt(s, smem_u32(sQ), aK);              // S = Q K^T
        mma_tt(dp, smem_u32(sdO), smem_u32(sV + st * TILE_BYTES));   // dP = dO V^T
        const int k0 = j * T;
        const bool edge = k0 + T - 1 > q0 + p.off || k0 + T > p.Sk;
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const int q = q0 + r0 + 8 * hh;
#pragma unroll
            for (int g = 0; g < 8; g++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int i = 4 * g + 2 * hh + e, key = k0 + 8 * g + cq + e;
                    const bool dead = edge && (key > q + p.off || key >= p.Sk);
                    const float pr = dead ? 0.f : exp2f(s[i] * sl2 - lse_r[hh]);
                    dp[i] = pr * (dp[i] - del_r[hh]);
                }
        }
        uint32_t pa[4][4];
        to_afrag(dp, pa);
        mma_pv(dqacc, pa, aK);                    // dQ += dS K
        __syncthreads();
    }
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        const int q = q0 + r0 + 8 * hh;
        if (q < p.Sq) {
            if (rope_cos) rope_bwd(dqacc, hh, rope_cos, rope_sin, q + p.off, cq);
            bf16* dst = dq + b * sdq.b + (long long)q * sdq.r + h * sdq.h + cq;
#pragma unroll
            for (int g = 0; g < 8; g++)
                *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack2(dqacc[4 * g + 2 * hh] * p.scale, dqacc[4 * g + 2 * hh + 1] * p.scale);
        }
    }
}

constexpr int SMEM_FWD = 5 * TILE_BYTES + 64 + 1024;
constexpr int SMEM_DKV = 6 * TILE_BYTES + 4 * T * 4 + 64 + 1024;
constexpr int SMEM_DQ = 6 * TILE_BYTES + 64 + 1024;

// tensor map of one operand: {n_heads * 64 columns, rows, batch}; heads must be contiguous 64-column blocks
int tmap_of(CUtensorMap* tm, const void* ptr, const long long* st, int n_heads, int rows, int batch, const char* what) {
    B200_CHECK_ARG(st[2] == D, "attn (wgmma): %s heads must be contiguous 64-column blocks (head stride %lld)", what, st[2]);
    B200_CHECK_ARG(st[1] % 8 == 0 && st[0] % 8 == 0 && (uintptr_t)ptr % 16 == 0,
                   "attn (wgmma): %s must be 16-byte aligned with row / batch strides a multiple of 8", what);
    return make_tmap_3d(tm, ptr, (uint64_t)n_heads * D, rows, batch, st[1], st[0], D, T);
}

template <typename K>
int set_smem(K kern, int bytes) {
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), "attn smem attr");
    return B200_OK;
}

}   // namespace

int b200_attn_bwd_delta_launch(const void* o, const void* d_o, float* delta, const long long* so, const long long* sdo,
                               int batch, int n_heads, int Sq, cudaStream_t stream);

// ===========================================================================
// C ABI: same contracts as b200_attn_causal_fwd / b200_attn_causal_bwd (attn_flash.cu); heads must be contiguous
// blocks of 64 columns (strides[.h] == 64).
// ===========================================================================
extern "C" int b200_attn_causal_fwd_wgmma(const void* q, const void* k, const void* v, void* o, float* lse,
                                          const long long* strides /* 4 x {b,r,h}: q,k,v,o */, int batch, int n_heads,
                                          int Sq, int Sk, int head_dim, float scale, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == D, "attn_causal_fwd_wgmma: head_dim %d unsupported (64 only)", head_dim);
    B200_CHECK_ARG(Sk >= Sq, "attn_causal_fwd_wgmma: Sk (%d) must be >= Sq (%d)", Sk, Sq);
    if (batch == 0 || Sq == 0) return B200_OK;
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tmap_of(&tq, q, strides, n_heads, Sq, batch, "q"))) return rc;
    if ((rc = tmap_of(&tk, k, strides + 3, n_heads, Sk, batch, "k"))) return rc;
    if ((rc = tmap_of(&tv, v, strides + 6, n_heads, Sk, batch, "v"))) return rc;
    static bool configured = false;
    if (!configured) {
        if ((rc = set_smem(attn_fwd_wgmma_kernel, SMEM_FWD))) return rc;
        configured = true;
    }
    const Strides so{strides[9], strides[10], strides[11]};
    const Params p{n_heads, Sq, Sk, Sk - Sq, scale};
    dim3 grid(batch * n_heads, (Sq + T - 1) / T);
    attn_fwd_wgmma_kernel<<<grid, NT, SMEM_FWD, stream>>>(tq, tk, tv, (bf16*)o, lse, so, p);
    B200_CHECK_LAUNCH("attn_causal_fwd_wgmma");
    return B200_OK;
}

extern "C" int b200_attn_causal_bwd_wgmma(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                          const float* lse, float* delta, void* dq, void* dk, void* dv,
                                          const long long* strides /* 8 x {b,r,h}: q,k,v,o,do,dq,dk,dv */, int batch,
                                          int n_heads, int Sq, int Sk, int head_dim, float scale, const void* rope_cos,
                                          const void* rope_sin, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == D, "attn_causal_bwd_wgmma: head_dim %d unsupported (64 only)", head_dim);
    B200_CHECK_ARG(Sk >= Sq, "attn_causal_bwd_wgmma: Sk must be >= Sq");
    if (batch == 0 || Sq == 0) return B200_OK;
    CUtensorMap tq, tk, tv, tdo;
    int rc;
    if ((rc = tmap_of(&tq, q, strides, n_heads, Sq, batch, "q"))) return rc;
    if ((rc = tmap_of(&tk, k, strides + 3, n_heads, Sk, batch, "k"))) return rc;
    if ((rc = tmap_of(&tv, v, strides + 6, n_heads, Sk, batch, "v"))) return rc;
    if ((rc = tmap_of(&tdo, d_o, strides + 12, n_heads, Sq, batch, "dO"))) return rc;
    if ((rc = b200_attn_bwd_delta_launch(o, d_o, delta, strides + 9, strides + 12, batch, n_heads, Sq, stream))) return rc;
    static bool configured = false;
    if (!configured) {
        if ((rc = set_smem(attn_bwd_dkv_wgmma_kernel, SMEM_DKV))) return rc;
        if ((rc = set_smem(attn_bwd_dq_wgmma_kernel, SMEM_DQ))) return rc;
        configured = true;
    }
    const Params p{n_heads, Sq, Sk, Sk - Sq, scale};
    const Strides sdq{strides[15], strides[16], strides[17]}, sdk{strides[18], strides[19], strides[20]},
        sdv{strides[21], strides[22], strides[23]};
    dim3 gkv(batch * n_heads, (Sk + T - 1) / T);
    attn_bwd_dkv_wgmma_kernel<<<gkv, NT, SMEM_DKV, stream>>>(tq, tk, tv, tdo, lse, delta, (bf16*)dk, (bf16*)dv, sdk, sdv, p,
                                                             (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_causal_bwd_dkv_wgmma");
    dim3 gq(batch * n_heads, (Sq + T - 1) / T);
    attn_bwd_dq_wgmma_kernel<<<gq, NT, SMEM_DQ, stream>>>(tq, tk, tv, tdo, lse, delta, (bf16*)dq, sdq, p,
                                                          (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_causal_bwd_dq_wgmma");
    return B200_OK;
}
