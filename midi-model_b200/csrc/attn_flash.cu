// Causal attention for the outer event stack (head_dim 64; hf sdpa_attention.py:92-101 called
// from modeling_llama.py:251-289 with is_causal=True, scale = d^-1/2), FlashAttention-style:
// online softmax in fp32, P rounded to bf16 for P.V, output rounded to bf16 (DESIGN.md 3.3).
//   fwd      : CTA = 64 query rows x (batch, head); K/V tiles of 64 keys double-buffered by cp.async
//   bwd dK/dV: CTA = 64 keys  x (batch, head), loops over query tiles      (no atomics, deterministic)
//   bwd dQ   : CTA = 64 query rows x (batch, head), loops over key tiles
// Tensor-core path here is mma.sync.m16n8k16 (bf16 -> fp32); operands are ldmatrix'ed from
// XOR-swizzled shared memory.  q/k/v are addressed through (batch, row, head) strides so the same
// kernels read the packed [rows, 3*hidden] qkv activation of training and the KV cache of prefill.
#include "common.cuh"
#include "rope.cuh"

namespace {

constexpr int D = 64;          // head_dim
constexpr int BM = 64;         // query rows per CTA
constexpr int BN = 64;         // keys per tile
constexpr int NT = 128;        // threads per CTA (4 warps x 16 rows)
constexpr float LOG2E = 1.4426950408889634f;

struct Strides {
    long long b, r, h;   // element strides: batch, row (position), head
};

// ---- primitives ----------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    const uint32_t s = smem_u32(smem);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A 64 x 64 bf16 tile in shared memory: row pitch 128 B, 16-byte chunk c of row r stored at chunk c ^ (r & 7).
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int row, int chunk) {
    return base + row * 128 + ((chunk ^ (row & 7)) << 4);
}

// Load a [64 rows x 64 cols] tile (rows row0.., zero-filled beyond n_rows) with cp.async.
__device__ __forceinline__ void load_tile(uint32_t sbase_generic_off, uint8_t* smem, const bf16* g, long long row_stride,
                                          int row0, int n_rows) {
    (void)sbase_generic_off;
#pragma unroll
    for (int i = 0; i < (64 * 8) / NT; i++) {
        const int idx = threadIdx.x + i * NT;
        const int r = idx >> 3, c = idx & 7;
        const bool ok = (row0 + r) < n_rows;
        const bf16* src = g + (long long)(ok ? row0 + r : 0) * row_stride + c * 8;
        cp_async16(smem + r * 128 + ((c ^ (r & 7)) << 4), src, ok);
    }
}

// A-operand fragments (16 rows x 64 k) for this warp's 16 rows starting at tile row `r0`.
__device__ __forceinline__ void load_a_frags(uint32_t sbase, int r0, uint32_t a[4][4]) {
    const int lane = threadIdx.x & 31;
    const int mat = lane >> 3, rr = lane & 7;
    const int row = r0 + rr + (mat & 1) * 8;
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
        const int chunk = kk * 2 + (mat >> 1);
        ldsm_x4(tile_addr(sbase, row, chunk), a[kk][0], a[kk][1], a[kk][2], a[kk][3]);
    }
}

// acc[nb][4] (16 x 64, nb = 8-column blocks) += A(16 x 64 over d) . T^T  where tile T is [n = 64 rows][k = 64 d].
__device__ __forceinline__ void mma_a_tileT(float acc[8][4], const uint32_t a[4][4], uint32_t sbase) {
    const int lane = threadIdx.x & 31;
    const int mat = lane >> 3, rr = lane & 7;
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
#pragma unroll
        for (int np = 0; np < 4; np++) {   // pairs of n-blocks
            const int row = np * 16 + (mat >> 1) * 8 + rr;
            const int chunk = kk * 2 + (mat & 1);
            uint32_t b0, b1, b2, b3;
            ldsm_x4(tile_addr(sbase, row, chunk), b0, b1, b2, b3);
            mma16816(acc[np * 2], a[kk], b0, b1);
            mma16816(acc[np * 2 + 1], a[kk], b2, b3);
        }
    }
}

// acc[nb][4] (16 x 64 over d) += P(16 x 64 over tile rows, as bf16 A fragments) . T  where tile T is [k = 64 rows][n = 64 d].
__device__ __forceinline__ void mma_p_tile(float acc[8][4], const uint32_t p[4][4], uint32_t sbase) {
    const int lane = threadIdx.x & 31;
    const int mat = lane >> 3, rr = lane & 7;
#pragma unroll
    for (int kb = 0; kb < 4; kb++) {
#pragma unroll
        for (int np = 0; np < 4; np++) {
            const int row = kb * 16 + (mat & 1) * 8 + rr;
            const int chunk = np * 2 + (mat >> 1);
            uint32_t b0, b1, b2, b3;
            ldsm_x4_t(tile_addr(sbase, row, chunk), b0, b1, b2, b3);
            mma16816(acc[np * 2], p[kb], b0, b1);
            mma16816(acc[np * 2 + 1], p[kb], b2, b3);
        }
    }
}

// accumulator (16 x 64 fp32) -> bf16 A fragments over its 64 columns
__device__ __forceinline__ void acc_to_afrag(const float s[8][4], uint32_t p[4][4]) {
#pragma unroll
    for (int kb = 0; kb < 4; kb++) {
        p[kb][0] = pack2(s[2 * kb][0], s[2 * kb][1]);
        p[kb][1] = pack2(s[2 * kb][2], s[2 * kb][3]);
        p[kb][2] = pack2(s[2 * kb + 1][0], s[2 * kb + 1][1]);
        p[kb][3] = pack2(s[2 * kb + 1][2], s[2 * kb + 1][3]);
    }
}

// ============================================================================================
// forward
// ============================================================================================
__global__ void __launch_bounds__(NT)
flash_fwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v, bf16* __restrict__ o,
                 float* __restrict__ lse, Strides sq, Strides sk, Strides sv, Strides so, int n_heads, int Sq, int Sk,
                 float scale) {
    __shared__ __align__(128) uint8_t smem[8192 * 5];   // Q | K0 | V0 | K1 | V1
    const int qt = gridDim.y - 1 - blockIdx.y;           // heavy (late) tiles first
    const int bh = blockIdx.x;
    const int b = bh / n_heads, h = bh % n_heads;
    const int off = Sk - Sq;
    const int q0 = qt * BM;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;

    const bf16* qg = q + b * sq.b + h * sq.h;
    const bf16* kg = k + b * sk.b + h * sk.h;
    const bf16* vg = v + b * sv.b + h * sv.h;
    const uint32_t sQ = smem_u32(smem);

    int n_kv = (min(q0 + BM - 1 + off, Sk - 1)) / BN + 1;
    if (n_kv < 1) n_kv = 1;

    load_tile(0, smem, qg, sq.r, q0, Sq);
    load_tile(0, smem + 8192, kg, sk.r, 0, Sk);
    load_tile(0, smem + 16384, vg, sv.r, 0, Sk);
    cp_async_commit();

    float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};
    float msc[2] = {0.f, 0.f};   // m_i * scale * log2(e), rounded once: every exponent of the row is taken against it
    float oacc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) oacc[i][j] = 0.f;
    uint32_t qa[4][4];
    const float sl2 = scale * LOG2E;

    for (int j = 0; j < n_kv; j++) {
        const int buf = j & 1;
        if (j + 1 < n_kv) {
            load_tile(0, smem + 8192 + (buf ^ 1) * 16384, kg, sk.r, (j + 1) * BN, Sk);
            load_tile(0, smem + 16384 + (buf ^ 1) * 16384, vg, sv.r, (j + 1) * BN, Sk);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (j == 0) load_a_frags(sQ, warp * 16, qa);
        const uint32_t sK = sQ + 8192 + buf * 16384, sV = sK + 8192;

        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int c = 0; c < 4; c++) s[i][c] = 0.f;
        mma_a_tileT(s, qa, sK);

        const int k0 = j * BN;
        const int row_a = q0 + warp * 16 + g;   // rows of c0,c1 ; row_a + 8 for c2,c3
        const bool need_mask = (k0 + BN - 1 > q0 + warp * 16 + off) || (k0 + BN > Sk);
        if (need_mask) {
#pragma unroll
            for (int nb = 0; nb < 8; nb++)
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int key = k0 + nb * 8 + 2 * t + (c & 1);
                    const int row = row_a + (c >> 1) * 8;
                    if (key > row + off || key >= Sk) s[nb][c] = -INFINITY;
                }
        }
        float mx[2] = {m_i[0], m_i[1]};
#pragma unroll
        for (int nb = 0; nb < 8; nb++) {
            mx[0] = fmaxf(mx[0], fmaxf(s[nb][0], s[nb][1]));
            mx[1] = fmaxf(mx[1], fmaxf(s[nb][2], s[nb][3]));
        }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
        float alpha[2], rs[2] = {0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const float mnew = mx[r];
            // The rescale is the difference of the old and new rounded reference points, so it is exactly 1 while the
            // max stays.  __fmul_rn keeps the product out of an FMA: m_old * sl2 - msc contracted to one FMA would be
            // 2^(rounding error of msc) instead, compounding over every key tile (1.9e-4 in the LSE at 64 tiles).
            const float ms = (mnew == -INFINITY) ? 0.f : __fmul_rn(mnew, sl2);
            alpha[r] = (m_i[r] == -INFINITY) ? 0.f : exp2f(msc[r] - ms);
            msc[r] = ms;
            m_i[r] = mnew;
        }
#pragma unroll
        for (int nb = 0; nb < 8; nb++) {
            s[nb][0] = exp2f(s[nb][0] * sl2 - msc[0]);
            s[nb][1] = exp2f(s[nb][1] * sl2 - msc[0]);
            s[nb][2] = exp2f(s[nb][2] * sl2 - msc[1]);
            s[nb][3] = exp2f(s[nb][3] * sl2 - msc[1]);
            rs[0] += s[nb][0] + s[nb][1];
            rs[1] += s[nb][2] + s[nb][3];
        }
#pragma unroll
        for (int r = 0; r < 2; r++) l_i[r] = l_i[r] * alpha[r] + rs[r];
#pragma unroll
        for (int nb = 0; nb < 8; nb++) {
            oacc[nb][0] *= alpha[0]; oacc[nb][1] *= alpha[0];
            oacc[nb][2] *= alpha[1]; oacc[nb][3] *= alpha[1];
        }
        uint32_t pa[4][4];
        acc_to_afrag(s, pa);
        mma_p_tile(oacc, pa, sV);
        __syncthreads();   // everyone done with buf before it is refilled two iterations later
    }

    // finalise: row sums across the quad, normalise, store
#pragma unroll
    for (int r = 0; r < 2; r++) {
        l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 1);
        l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 2);
    }
    bf16* og = o + b * so.b + h * so.h;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int row = q0 + warp * 16 + g + r * 8;
        if (row < Sq) {
            const float inv = l_i[r] > 0.f ? 1.f / l_i[r] : 0.f;
#pragma unroll
            for (int nb = 0; nb < 8; nb++) {
                *reinterpret_cast<uint32_t*>(og + (long long)row * so.r + nb * 8 + 2 * t) =
                    pack2(oacc[nb][2 * r] * inv, oacc[nb][2 * r + 1] * inv);
            }
            if (t == 0 && lse) lse[((long long)b * n_heads + h) * Sq + row] = m_i[r] * scale + logf(l_i[r]);
        }
    }
}

// ============================================================================================
// backward
// ============================================================================================
// Optional fused RoPE backward: the gradient w.r.t. the *pre-rotation* q / k, on the accumulators; the (d, d+32) pairs
// are accumulator blocks (nb, nb+4) of the same thread.
__device__ __forceinline__ void rope_bwd_acc(float acc[8][4], int r, const bf16* __restrict__ cos_t,
                                             const bf16* __restrict__ sin_t, int pos, int t) {
#pragma unroll
    for (int nb = 0; nb < 4; nb++) {
        const float2 c = __bfloat1622float2(*reinterpret_cast<const bf162*>(cos_t + (size_t)pos * 32 + nb * 8 + 2 * t));
        const float2 sn = __bfloat1622float2(*reinterpret_cast<const bf162*>(sin_t + (size_t)pos * 32 + nb * 8 + 2 * t));
        const float a0 = acc[nb][2 * r], a1 = acc[nb][2 * r + 1];
        const float b0 = acc[nb + 4][2 * r], b1 = acc[nb + 4][2 * r + 1];
        acc[nb][2 * r] = rope_bwd_elem(a0, b0, c.x, sn.x, false);
        acc[nb][2 * r + 1] = rope_bwd_elem(a1, b1, c.y, sn.y, false);
        acc[nb + 4][2 * r] = rope_bwd_elem(b0, a0, c.x, sn.x, true);
        acc[nb + 4][2 * r + 1] = rope_bwd_elem(b1, a1, c.y, sn.y, true);
    }
}

// delta[b,h,q] = sum_d dO[q,d] * O[q,d]; one 128-thread CTA per (b, q) row of n_heads*64 columns
__global__ void flash_bwd_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, float* __restrict__ delta,
                                       Strides so, Strides sdo, int n_heads, int Sq) {
    const int row = blockIdx.x % Sq, b = blockIdx.x / Sq;
    // whole warps stay in the loop (full-mask shuffles); lanes past the last head contribute nothing
    for (int i0 = 0; i0 < n_heads * 8; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x, h = i >> 3, c = i & 7;
        float s = 0.f;
        if (h < n_heads) {
            float a[8], d[8];
            unpack8(*reinterpret_cast<const uint4*>(o + b * so.b + (long long)row * so.r + h * so.h + c * 8), a);
            unpack8(*reinterpret_cast<const uint4*>(d_o + b * sdo.b + (long long)row * sdo.r + h * sdo.h + c * 8), d);
#pragma unroll
            for (int j = 0; j < 8; j++) s += a[j] * d[j];
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        if (h < n_heads && c == 0) delta[((long long)b * n_heads + h) * Sq + row] = s;
    }
}

// dK, dV for one tile of 64 keys: S^T = K Q^T (rows = keys), loops over query tiles
__global__ void __launch_bounds__(NT, 3)
flash_bwd_dkv_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                     const bf16* __restrict__ d_o, const float* __restrict__ lse, const float* __restrict__ delta,
                     bf16* __restrict__ dk, bf16* __restrict__ dv, Strides sq, Strides sk, Strides sv, Strides sdo,
                     Strides sdk, Strides sdv, int n_heads, int Sq, int Sk, float scale, const bf16* __restrict__ rope_cos,
                     const bf16* __restrict__ rope_sin) {
    extern __shared__ __align__(128) uint8_t smem[];    // K | V | Q0 | dO0 | Q1 | dO1 | lse[2][64] | delta[2][64]
    float (*s_lse)[BM] = reinterpret_cast<float (*)[BM]>(smem + 8192 * 6);
    float (*s_delta)[BM] = reinterpret_cast<float (*)[BM]>(smem + 8192 * 6 + 2 * BM * 4);
    const int kt = blockIdx.y;       // slow grid index: all heavy (early-key) tiles are scheduled first
    const int bh = blockIdx.x;
    const int b = bh / n_heads, h = bh % n_heads;
    const int off = Sk - Sq;
    const int k0 = kt * BN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;

    const bf16* qg = q + b * sq.b + h * sq.h;
    const bf16* kg = k + b * sk.b + h * sk.h;
    const bf16* vg = v + b * sv.b + h * sv.h;
    const bf16* dog = d_o + b * sdo.b + h * sdo.h;
    const float* lse_g = lse + ((long long)b * n_heads + h) * Sq;
    const float* delta_g = delta + ((long long)b * n_heads + h) * Sq;
    const uint32_t sK = smem_u32(smem), sV = sK + 8192;

    int qt0 = (k0 - off) / BM;
    if (k0 - off < 0) qt0 = 0;
    const int n_qt = (Sq + BM - 1) / BM;

    float dkacc[8][4], dvacc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int c = 0; c < 4; c++) { dkacc[i][c] = 0.f; dvacc[i][c] = 0.f; }

    load_tile(0, smem, kg, sk.r, k0, Sk);
    load_tile(0, smem + 8192, vg, sv.r, k0, Sk);
    if (qt0 < n_qt) {
        load_tile(0, smem + 16384, qg, sq.r, qt0 * BM, Sq);
        load_tile(0, smem + 24576, dog, sdo.r, qt0 * BM, Sq);
        if (threadIdx.x < BM) {
            const int r = qt0 * BM + threadIdx.x;
            s_lse[0][threadIdx.x] = r < Sq ? lse_g[r] : 0.f;
            s_delta[0][threadIdx.x] = r < Sq ? delta_g[r] : 0.f;
        }
    }
    cp_async_commit();
    uint32_t ka[4][4], va[4][4];
    const float sl2 = scale * LOG2E;

    for (int qt = qt0; qt < n_qt; qt++) {
        const int buf = (qt - qt0) & 1;
        if (qt + 1 < n_qt) {
            load_tile(0, smem + 16384 + (buf ^ 1) * 16384, qg, sq.r, (qt + 1) * BM, Sq);
            load_tile(0, smem + 24576 + (buf ^ 1) * 16384, dog, sdo.r, (qt + 1) * BM, Sq);
            if (threadIdx.x < BM) {
                const int r = (qt + 1) * BM + threadIdx.x;
                s_lse[buf ^ 1][threadIdx.x] = r < Sq ? lse_g[r] : 0.f;
                s_delta[buf ^ 1][threadIdx.x] = r < Sq ? delta_g[r] : 0.f;
            }
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (qt == qt0) {
            load_a_frags(sK, warp * 16, ka);
            load_a_frags(sV, warp * 16, va);
        }
        const uint32_t sQ = sK + 16384 + buf * 16384, sDO = sQ + 8192;
        const int q0 = qt * BM;

        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int c = 0; c < 4; c++) s[i][c] = 0.f;
        mma_a_tileT(s, ka, sQ);   // S^T[key, q]
        const int key_a = k0 + warp * 16 + g;
#pragma unroll
        for (int nb = 0; nb < 8; nb++)
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int qq = nb * 8 + 2 * t + (c & 1);
                const int key = key_a + (c >> 1) * 8;
                const int qrow = q0 + qq;
                const bool dead = (key > qrow + off) || (key >= Sk) || (qrow >= Sq);
                s[nb][c] = dead ? 0.f : exp2f(s[nb][c] * sl2 - s_lse[buf][qq] * LOG2E);
            }
        float dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int c = 0; c < 4; c++) dp[i][c] = 0.f;
        mma_a_tileT(dp, va, sDO);   // dP^T[key, q] = V dO^T
        uint32_t pa[4][4];
        acc_to_afrag(s, pa);
        mma_p_tile(dvacc, pa, sDO);   // dV += P^T dO
#pragma unroll
        for (int nb = 0; nb < 8; nb++)
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int qq = nb * 8 + 2 * t + (c & 1);
                dp[nb][c] = s[nb][c] * (dp[nb][c] - s_delta[buf][qq]);
            }
        acc_to_afrag(dp, pa);
        mma_p_tile(dkacc, pa, sQ);    // dK += dS^T Q
        __syncthreads();
    }

    bf16* dkg = dk + b * sdk.b + h * sdk.h;
    bf16* dvg = dv + b * sdv.b + h * sdv.h;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int key = k0 + warp * 16 + g + r * 8;
        if (key < Sk) {
            if (rope_cos) rope_bwd_acc(dkacc, r, rope_cos, rope_sin, key, t);   // linear: commutes with the scale below
#pragma unroll
            for (int nb = 0; nb < 8; nb++) {
                *reinterpret_cast<uint32_t*>(dkg + (long long)key * sdk.r + nb * 8 + 2 * t) =
                    pack2(dkacc[nb][2 * r] * scale, dkacc[nb][2 * r + 1] * scale);
                *reinterpret_cast<uint32_t*>(dvg + (long long)key * sdv.r + nb * 8 + 2 * t) =
                    pack2(dvacc[nb][2 * r], dvacc[nb][2 * r + 1]);
            }
        }
    }
}

// dQ for one tile of 64 query rows, loops over key tiles
__global__ void __launch_bounds__(NT, 3)
flash_bwd_dq_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                    const bf16* __restrict__ d_o, const float* __restrict__ lse, const float* __restrict__ delta,
                    bf16* __restrict__ dq, Strides sq, Strides sk, Strides sv, Strides sdo, Strides sdq, int n_heads,
                    int Sq, int Sk, float scale, const bf16* __restrict__ rope_cos, const bf16* __restrict__ rope_sin) {
    extern __shared__ __align__(128) uint8_t smem[];    // Q | dO | K0 | V0 | K1 | V1
    const int qt = gridDim.y - 1 - blockIdx.y;
    const int bh = blockIdx.x;
    const int b = bh / n_heads, h = bh % n_heads;
    const int off = Sk - Sq;
    const int q0 = qt * BM;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;

    const bf16* qg = q + b * sq.b + h * sq.h;
    const bf16* kg = k + b * sk.b + h * sk.h;
    const bf16* vg = v + b * sv.b + h * sv.h;
    const bf16* dog = d_o + b * sdo.b + h * sdo.h;
    const uint32_t sQ = smem_u32(smem), sDO = sQ + 8192;

    int n_kv = (min(q0 + BM - 1 + off, Sk - 1)) / BN + 1;
    if (n_kv < 1) n_kv = 1;

    load_tile(0, smem, qg, sq.r, q0, Sq);
    load_tile(0, smem + 8192, dog, sdo.r, q0, Sq);
    load_tile(0, smem + 16384, kg, sk.r, 0, Sk);
    load_tile(0, smem + 24576, vg, sv.r, 0, Sk);
    cp_async_commit();

    float lse_r[2], delta_r[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int row = q0 + warp * 16 + g + r * 8;
        const long long idx = ((long long)b * n_heads + h) * Sq + row;
        lse_r[r] = row < Sq ? lse[idx] * LOG2E : 0.f;
        delta_r[r] = row < Sq ? delta[idx] : 0.f;
    }
    float dqacc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int c = 0; c < 4; c++) dqacc[i][c] = 0.f;
    uint32_t qa[4][4], doa[4][4];
    const float sl2 = scale * LOG2E;

    for (int j = 0; j < n_kv; j++) {
        const int buf = j & 1;
        if (j + 1 < n_kv) {
            load_tile(0, smem + 16384 + (buf ^ 1) * 16384, kg, sk.r, (j + 1) * BN, Sk);
            load_tile(0, smem + 24576 + (buf ^ 1) * 16384, vg, sv.r, (j + 1) * BN, Sk);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (j == 0) {
            load_a_frags(sQ, warp * 16, qa);
            load_a_frags(sDO, warp * 16, doa);
        }
        const uint32_t sK = sQ + 16384 + buf * 16384, sV = sK + 8192;
        const int k0 = j * BN;

        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int c = 0; c < 4; c++) s[i][c] = 0.f;
        mma_a_tileT(s, qa, sK);
        const int row_a = q0 + warp * 16 + g;
#pragma unroll
        for (int nb = 0; nb < 8; nb++)
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int key = k0 + nb * 8 + 2 * t + (c & 1);
                const int row = row_a + (c >> 1) * 8;
                const bool dead = (key > row + off) || (key >= Sk) || (row >= Sq);
                s[nb][c] = dead ? 0.f : exp2f(s[nb][c] * sl2 - lse_r[c >> 1]);
            }
        float dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int c = 0; c < 4; c++) dp[i][c] = 0.f;
        mma_a_tileT(dp, doa, sV);   // dP = dO V^T
#pragma unroll
        for (int nb = 0; nb < 8; nb++)
#pragma unroll
            for (int c = 0; c < 4; c++) dp[nb][c] = s[nb][c] * (dp[nb][c] - delta_r[c >> 1]);
        uint32_t pa[4][4];
        acc_to_afrag(dp, pa);
        mma_p_tile(dqacc, pa, sK);   // dQ += dS K
        __syncthreads();
    }

    bf16* dqg = dq + b * sdq.b + h * sdq.h;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int row = q0 + warp * 16 + g + r * 8;
        if (row < Sq) {
            if (rope_cos) rope_bwd_acc(dqacc, r, rope_cos, rope_sin, row + off, t);
#pragma unroll
            for (int nb = 0; nb < 8; nb++)
                *reinterpret_cast<uint32_t*>(dqg + (long long)row * sdq.r + nb * 8 + 2 * t) =
                    pack2(dqacc[nb][2 * r] * scale, dqacc[nb][2 * r + 1] * scale);
        }
    }
}

}   // namespace

// ===========================================================================
// C ABI.  Strides are element strides {batch, row, head}; head_dim is fixed at 64.
// ===========================================================================
extern "C" int b200_attn_causal_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                                    const long long* strides /* 4 x {b,r,h}: q,k,v,o */, int batch, int n_heads, int Sq,
                                    int Sk, int head_dim, float scale, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == D, "attn_causal_fwd: head_dim %d unsupported (64 only)", head_dim);
    B200_CHECK_ARG(Sk >= Sq, "attn_causal_fwd: Sk (%d) must be >= Sq (%d)", Sk, Sq);
    if (batch == 0 || Sq == 0) return B200_OK;
    Strides s[4];
    for (int i = 0; i < 4; i++) { s[i].b = strides[3 * i]; s[i].r = strides[3 * i + 1]; s[i].h = strides[3 * i + 2]; }
    static bool configured = false;
    if (!configured) {   // let 4+ CTAs (40 KB static smem each) share an SM
        B200_CUDA(cudaFuncSetAttribute(flash_fwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared), "attn carveout");
        configured = true;
    }
    dim3 grid(batch * n_heads, (Sq + BM - 1) / BM);   // tiles on the slow index: longest first across all heads
    flash_fwd_kernel<<<grid, NT, 0, stream>>>((const bf16*)q, (const bf16*)k, (const bf16*)v, (bf16*)o, lse, s[0], s[1],
                                             s[2], s[3], n_heads, Sq, Sk, scale);
    B200_CHECK_LAUNCH("attn_causal_fwd");
    return B200_OK;
}

// delta[b,h,q] = rowsum(dO * O)
int b200_attn_bwd_delta_launch(const void* o, const void* d_o, float* delta, const long long* so, const long long* sdo,
                               int batch, int n_heads, int Sq, cudaStream_t stream) {
    Strides a{so[0], so[1], so[2]}, b{sdo[0], sdo[1], sdo[2]};
    flash_bwd_delta_kernel<<<batch * Sq, 128, 0, stream>>>((const bf16*)o, (const bf16*)d_o, delta, a, b, n_heads, Sq);
    B200_CHECK_LAUNCH("attn_bwd_delta");
    return B200_OK;
}

// delta: float[batch*n_heads*Sq] workspace
extern "C" int b200_attn_causal_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                    const float* lse, float* delta, void* dq, void* dk, void* dv,
                                    const long long* strides /* 8 x {b,r,h}: q,k,v,o,do,dq,dk,dv */, int batch,
                                    int n_heads, int Sq, int Sk, int head_dim, float scale, const void* rope_cos,
                                    const void* rope_sin, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == D, "attn_causal_bwd: head_dim %d unsupported (64 only)", head_dim);
    B200_CHECK_ARG(Sk >= Sq, "attn_causal_bwd: Sk must be >= Sq");
    if (batch == 0 || Sq == 0) return B200_OK;
    Strides s[8];
    for (int i = 0; i < 8; i++) { s[i].b = strides[3 * i]; s[i].r = strides[3 * i + 1]; s[i].h = strides[3 * i + 2]; }
    flash_bwd_delta_kernel<<<batch * Sq, 128, 0, stream>>>((const bf16*)o, (const bf16*)d_o, delta, s[3], s[4], n_heads, Sq);
    B200_CHECK_LAUNCH("attn_causal_bwd_delta");
    B200_CHECK_ARG(n_heads % 4 == 0, "attn_causal_bwd: n_heads must be a multiple of 4");
    constexpr int SMEM_BWD = 8192 * 6 + 4 * BM * 4;
    static bool configured = false;
    if (!configured) {
        B200_CUDA(cudaFuncSetAttribute(flash_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BWD), "attn smem");
        B200_CUDA(cudaFuncSetAttribute(flash_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BWD), "attn smem");
        B200_CUDA(cudaFuncSetAttribute(flash_bwd_dkv_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared), "attn carveout");
        B200_CUDA(cudaFuncSetAttribute(flash_bwd_dq_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared), "attn carveout");
        configured = true;
    }
    dim3 gkv(batch * n_heads, (Sk + BN - 1) / BN);   // tiles on the slow index: longest first across all heads
    flash_bwd_dkv_kernel<<<gkv, NT, SMEM_BWD, stream>>>((const bf16*)q, (const bf16*)k, (const bf16*)v, (const bf16*)d_o, lse, delta,
                                                 (bf16*)dk, (bf16*)dv, s[0], s[1], s[2], s[4], s[6], s[7], n_heads, Sq, Sk,
                                                 scale, (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_causal_bwd_dkv");
    dim3 gq(batch * n_heads, (Sq + BM - 1) / BM);   // tiles on the slow index: longest first across all heads
    flash_bwd_dq_kernel<<<gq, NT, SMEM_BWD, stream>>>((const bf16*)q, (const bf16*)k, (const bf16*)v, (const bf16*)d_o, lse, delta,
                                               (bf16*)dq, s[0], s[1], s[2], s[4], s[5], n_heads, Sq, Sk, scale,
                                               (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_causal_bwd_dq");
    return B200_OK;
}
