// Kernels of the generate() loop (midi_model.py:167-250): every step is a handful of rows, so
// all of this is HBM-bound weight / KV streaming.
//  * skinny GEMM  y[B<=16, N] = x . W^T     -- one warp per output column streams the weight row
//    with 16-byte loads, activations staged in shared memory, fp32 accumulate (nn.Linear rounding)
//  * paged KV cache (pages of PAGE positions, per-row block table): append + single-query attention
//    with split-T partials and a combine pass (replaces DynamicCache's torch.cat, hf cache_utils.py:119)
//  * fused sampler: temperature, full-vocab softmax, grammar range / mask, top-p, top-k, draw
//    (midi_model.py:222-223 + 152-165), one CTA per row, bitonic sort of the non-zero entries only.
#include "common.cuh"
#include "rope.cuh"
#include "sampler.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// skinny GEMM
// ---------------------------------------------------------------------------------------------
constexpr int GV_WARPS = 8;

// Plain skinny GEMM (b200_gemv_bf16).  gemv_fused_kernel without its options gives the same bits, but it stages x one
// warp per row and holds 70-80 registers: through it, 1-3 rows and the vocabulary projection ran up to 1.5x slower
// (profiles/h100_decode_ab.txt), so both kernels stay.
template <int B>
__global__ void __launch_bounds__(GV_WARPS * 32)
gemv_kernel(const bf16* __restrict__ x, const bf16* __restrict__ W, const bf16* __restrict__ res, bf16* __restrict__ y,
            int N, int K, int ldx, int ldw, int ldr, int ldy) {
    extern __shared__ __align__(16) uint8_t gv_smem[];
    bf16* xs = reinterpret_cast<bf16*>(gv_smem);   // [B][K]
    const int nvec = K / 8;
    for (int i = threadIdx.x; i < B * nvec; i += blockDim.x) {
        const int b = i / nvec, v = i % nvec;
        *reinterpret_cast<uint4*>(xs + b * K + v * 8) = *reinterpret_cast<const uint4*>(x + (size_t)b * ldx + v * 8);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int n = blockIdx.x * GV_WARPS + warp; n < N; n += gridDim.x * GV_WARPS) {
        float acc[B];
#pragma unroll
        for (int b = 0; b < B; b++) acc[b] = 0.f;
        const bf16* wrow = W + (size_t)n * ldw;
        for (int v = lane; v < nvec; v += 32) {
            float wf[8];
            unpack8(ld_nc16(wrow + v * 8), wf);
#pragma unroll
            for (int b = 0; b < B; b++) {
                float xf[8];
                unpack8(*reinterpret_cast<const uint4*>(xs + b * K + v * 8), xf);
#pragma unroll
                for (int j = 0; j < 8; j++) acc[b] = fmaf(wf[j], xf[j], acc[b]);
            }
        }
#pragma unroll
        for (int b = 0; b < B; b++) acc[b] = warp_sum(acc[b]);
        if (lane == 0) {
#pragma unroll
            for (int b = 0; b < B; b++) {
                float o = acc[b];
                if (res) o = bf16_round(o) + __bfloat162float(res[(size_t)b * ldr + n]);
                y[(size_t)b * ldy + n] = __float2bfloat16_rn(o);
            }
        }
    }
}

// Fused decode-step projection: y = [swiglu]( [rmsnorm_w](x) . W^T ) [+ res]
//   * x rows come from `x` or are gathered from an embedding table (`ids` != NULL: row b = table[ids[b * ids_stride]],
//     midi_model.py:128 -- the token-level stack's input at steps 1..7)
//   * norm_w != NULL : RMSNorm (hf :62-67, two roundings) applied while staging x in shared memory
//   * swiglu != 0    : W = [gate | up] rows, output n = bf16(bf16(silu(g_n)) * u_n) with g, u = bf16(acc)  (hf :183)
// Same rounding points as the stand-alone kernels, so fused and unfused decode are bit-identical.
template <int B>
__global__ void __launch_bounds__(GV_WARPS * 32)
gemv_fused_kernel(const bf16* __restrict__ x, const long long* __restrict__ ids, int ids_stride, const bf16* __restrict__ table,
                  const bf16* __restrict__ norm_w, float eps, const bf16* __restrict__ W, const bf16* __restrict__ res,
                  bf16* __restrict__ y, int N_out, int K, int ldx, int ldw, int ldr, int ldy, int swiglu, int V) {
    extern __shared__ __align__(16) uint8_t gv_smem[];
    bf16* xs = reinterpret_cast<bf16*>(gv_smem);   // [B][K]
    const int nvec = K / 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // prefetch this warp's first weight row (up to 4 vectors per lane) BEFORE staging x: the DRAM latency of the weights
    // then overlaps the x load / RMSNorm prologue instead of following it
    constexpr int PF = 4;
    uint4 wpre[PF] = {}, wpre2[PF] = {};
    const int n_first = blockIdx.x * GV_WARPS + warp;
    if (n_first < N_out) {
#pragma unroll
        for (int i = 0; i < PF; i++) {
            const int v = lane + i * 32;
            if (v < nvec) {
                wpre[i] = ld_nc16(W + (size_t)n_first * ldw + v * 8);
                if (swiglu) wpre2[i] = ld_nc16(W + (size_t)(n_first + N_out) * ldw + v * 8);
            }
        }
    }
    for (int b = warp; b < B; b += GV_WARPS) {     // one warp stages (and normalises) one row
        const bf16* src;
        if (ids) {
            long long id = ids[(size_t)b * ids_stride];
            if (id < 0 || id >= V) id = 0;
            src = table + (size_t)id * K;
        } else {
            src = x + (size_t)b * ldx;
        }
        if (norm_w) {
            float ss = 0.f;
            for (int v = lane; v < nvec; v += 32) {
                float f[8];
                unpack8(*reinterpret_cast<const uint4*>(src + v * 8), f);
#pragma unroll
                for (int j = 0; j < 8; j++) ss = fmaf(f[j], f[j], ss);
            }
            ss = warp_sum(ss);
            const float rstd = rsqrtf(ss / (float)K + eps);
            for (int v = lane; v < nvec; v += 32) {
                float f[8], wv[8];
                unpack8(*reinterpret_cast<const uint4*>(src + v * 8), f);
                unpack8(*reinterpret_cast<const uint4*>(norm_w + v * 8), wv);
#pragma unroll
                for (int j = 0; j < 8; j++) f[j] = wv[j] * bf16_round(f[j] * rstd);
                *reinterpret_cast<uint4*>(xs + b * K + v * 8) = pack8(f);
            }
        } else {
            for (int v = lane; v < nvec; v += 32)
                *reinterpret_cast<uint4*>(xs + b * K + v * 8) = *reinterpret_cast<const uint4*>(src + v * 8);
        }
    }
    __syncthreads();
    for (int n = blockIdx.x * GV_WARPS + warp; n < N_out; n += gridDim.x * GV_WARPS) {
        float acc[B], acc2[B];
#pragma unroll
        for (int b = 0; b < B; b++) { acc[b] = 0.f; acc2[b] = 0.f; }
        const bf16* wrow = W + (size_t)n * ldw;
        const bf16* wrow2 = W + (size_t)(n + N_out) * ldw;     // "up" row when swiglu
        const bool first = (n == n_first);
        auto accumulate = [&](const uint4& w1, const uint4& w2, int v) {
            float wf[8], wf2[8];
            unpack8(w1, wf);
            if (swiglu) unpack8(w2, wf2);
#pragma unroll
            for (int b = 0; b < B; b++) {
                float xf[8];
                unpack8(*reinterpret_cast<const uint4*>(xs + b * K + v * 8), xf);
#pragma unroll
                for (int j = 0; j < 8; j++) acc[b] = fmaf(wf[j], xf[j], acc[b]);
                if (swiglu) {
#pragma unroll
                    for (int j = 0; j < 8; j++) acc2[b] = fmaf(wf2[j], xf[j], acc2[b]);
                }
            }
        };
#pragma unroll
        for (int i = 0; i < PF; i++) {               // vectors covered by the prefetch registers (static indexing)
            const int v = lane + i * 32;
            if (v < nvec) {
                uint4 w1 = wpre[i], w2 = wpre2[i];
                if (!first) {
                    w1 = ld_nc16(wrow + v * 8);
                    if (swiglu) w2 = ld_nc16(wrow2 + v * 8);
                }
                accumulate(w1, w2, v);
            }
        }
        for (int v = lane + PF * 32; v < nvec; v += 32) {
            const uint4 w1 = ld_nc16(wrow + v * 8);
            uint4 w2 = w1;
            if (swiglu) w2 = ld_nc16(wrow2 + v * 8);
            accumulate(w1, w2, v);
        }
#pragma unroll
        for (int b = 0; b < B; b++) {
            acc[b] = warp_sum(acc[b]);
            if (swiglu) acc2[b] = warp_sum(acc2[b]);
        }
        if (lane == 0) {
#pragma unroll
            for (int b = 0; b < B; b++) {
                float o = acc[b];
                if (swiglu) {
                    const float g = bf16_round(o), u = bf16_round(acc2[b]);
                    o = bf16_round(silu_f(g)) * u;
                }
                if (res) o = bf16_round(o) + __bfloat162float(res[(size_t)b * ldr + n]);
                y[(size_t)b * ldy + n] = __float2bfloat16_rn(o);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// paged KV cache
// ---------------------------------------------------------------------------------------------
struct KVLayout {
    bf16* k_pool;          // [n_pages][n_heads][page][D]
    bf16* v_pool;
    const int* block_table;   // [batch][max_pages]
    int max_pages, page, n_heads, D;
};
__device__ __forceinline__ size_t kv_off(const KVLayout& L, int b, int h, int t) {
    const int pg = L.block_table[b * L.max_pages + t / L.page];
    return (((size_t)pg * L.n_heads + h) * L.page + (t % L.page)) * L.D;
}

// copy the k / v thirds of packed qkv rows [batch*s_new, 3H] into the cache at positions pos0 .. pos0+s_new-1
// (RAGGED: row b's at pos0 + row_off[b] ..)
template <bool RAGGED>
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, KVLayout L, int s_new, int pos0, const int* pos0_dev, int ld,
                                 const int* __restrict__ row_off) {
    const int r = blockIdx.x;
    const int b = r / s_new, i = r % s_new;
    int t = (pos0_dev ? *pos0_dev : pos0) + i;
    if constexpr (RAGGED) t += row_off[b];
    const int H = L.n_heads * L.D;
    const int vec_per_head = L.D / 8;
    for (int c = threadIdx.x; c < H / 8; c += blockDim.x) {
        const int h = c / vec_per_head, dv = c % vec_per_head;
        const size_t o = kv_off(L, b, h, t) + dv * 8;
        *reinterpret_cast<uint4*>(L.k_pool + o) = *reinterpret_cast<const uint4*>(qkv + (size_t)r * ld + H + c * 8);
        *reinterpret_cast<uint4*>(L.v_pool + o) = *reinterpret_cast<const uint4*>(qkv + (size_t)r * ld + 2 * H + c * 8);
    }
}

// K / V rows of one (batch row, head) in the cache; K is read through the non-coherent, L1-bypassing path
struct CacheRows {
    KVLayout L;
    int b, h;
    __device__ __forceinline__ const bf16* key(int t) const { return L.k_pool + kv_off(L, b, h, t); }
    __device__ __forceinline__ const bf16* value(int t) const { return L.v_pool + kv_off(L, b, h, t); }
    __device__ __forceinline__ void unpack_key8(const bf16* p, float* f) const { unpack8(ld_nc16(p), f); }
};
// the same, except that position `pos` comes from shared memory (the kernel appends it to the cache itself), so K is
// read with generic loads
struct CacheRowsWithNew {
    CacheRows cache;
    const bf16* s_k;
    const bf16* s_v;
    int pos;
    __device__ __forceinline__ const bf16* key(int t) const { return t == pos ? s_k : cache.key(t); }
    __device__ __forceinline__ const bf16* value(int t) const { return t == pos ? s_v : cache.value(t); }
    __device__ __forceinline__ void unpack_key8(const bf16* p, float* f) const {
        unpack8(*reinterpret_cast<const uint4*>(p), f);
    }
};

// partial record of a split with no keys: it drops out of the combine pass
template <int D>
__device__ __forceinline__ void write_empty_partial(float* pout) {
    if (threadIdx.x == 0) { pout[0] = -INFINITY; pout[1] = 0.f; }
    for (int d = threadIdx.x; d < D; d += blockDim.x) pout[2 + d] = 0.f;
}

// Single-query attention of q (in shared memory) over keys [t0, t1), t0 < t1, by one 128-thread CTA.  Writes the partial
// record pout = (m, l, o[D]) for the combine pass or, when `direct` (the chunk is the whole context), the normalised
// output row out_row()[0..D).  out_row is called only then: an output address formed up front would hold registers
// through the key loops and cut the loads ptxas keeps in flight there.
template <int D, typename Rows, typename OutRow>
__device__ __forceinline__ void attend_chunk(const bf16* s_q, const Rows& rows, int t0, int t1, float scale, float* pout,
                                             bool direct, OutRow out_row) {
    constexpr int CHUNK_MAX = 1024;
    __shared__ float s_sc[CHUNK_MAX];
    __shared__ float s_red[8];
    __shared__ float s_out[2][D];
    // scores: one thread per key
    float mx = -INFINITY;
    for (int t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
        const bf16* kp = rows.key(t);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < D / 8; d++) {
            float kf[8], qf[8];
            rows.unpack_key8(kp + d * 8, kf);
            unpack8(*reinterpret_cast<const uint4*>(s_q + d * 8), qf);
#pragma unroll
            for (int j = 0; j < 8; j++) s = fmaf(kf[j], qf[j], s);
        }
        s *= scale;
        s_sc[t - t0] = s;
        mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(s_red[0], s_red[1]), fmaxf(s_red[2], s_red[3]));
    float sum = 0.f;
    for (int t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
        const float p = __expf(s_sc[t - t0] - mx);
        sum += p;
        s_sc[t - t0] = bf16_round(p);   // P rounded to bf16 before P.V (flash semantics)
    }
    sum = warp_sum(sum);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[4 + (threadIdx.x >> 5)] = sum;
    __syncthreads();
    sum = s_red[4] + s_red[5] + s_red[6] + s_red[7];
    // output: threads split (key parity group, d)
    constexpr int GROUPS = (D >= 128) ? 1 : 128 / D;   // D=64 -> 2 groups of 64 threads ; D=256 -> 1 group, 2 d per thread
    constexpr int DPT = (D >= 128) ? D / 128 : 1;
    const int grp = (D >= 128) ? 0 : threadIdx.x / D;
    const int d0 = (D >= 128) ? threadIdx.x * DPT : threadIdx.x % D;
    float acc[DPT];
#pragma unroll
    for (int j = 0; j < DPT; j++) acc[j] = 0.f;
    for (int t = t0 + grp; t < t1; t += GROUPS) {
        const bf16* vp = rows.value(t);
        const float p = s_sc[t - t0];
#pragma unroll
        for (int j = 0; j < DPT; j++) acc[j] = fmaf(p, __bfloat162float(vp[d0 + j]), acc[j]);
    }
    if (GROUPS == 2) {
        s_out[grp][d0] = acc[0];
        __syncthreads();
        acc[0] = s_out[0][d0] + s_out[1][d0];
    }
    if (direct) {
        bf16* out = out_row();
        if (grp == 0) {
#pragma unroll
            for (int j = 0; j < DPT; j++) out[d0 + j] = __float2bfloat16_rn(acc[j] / sum);
        }
    } else {
        if (grp == 0) {
#pragma unroll
            for (int j = 0; j < DPT; j++) pout[2 + d0 + j] = acc[j];
        }
        if (threadIdx.x == 0) { pout[0] = mx; pout[1] = sum; }
    }
}

// single-query attention over the cache.  Row r = b * s_q + i attends to keys 0 .. past + i (RAGGED: past + row_off[b] + i).
// grid (rows * n_heads, n_split); partial: [rows*n_heads][n_split][D + 2] = (m, l, o[D])
template <int D, bool RAGGED>
__global__ void __launch_bounds__(128)
decode_attn_kernel(const bf16* __restrict__ q, KVLayout L, float* __restrict__ partial, int s_q, int past,
                   const int* past_dev, int ldq, float scale, int n_split, const int* __restrict__ row_off) {
    __shared__ __align__(16) bf16 s_q_sh[D];
    const int rh = blockIdx.x;
    const int r = rh / L.n_heads, h = rh % L.n_heads;
    const int b = r / s_q, i = r % s_q;
    int T = (past_dev ? *past_dev : past) + i + 1;
    if constexpr (RAGGED) T += row_off[b];
    const int chunk = (T + n_split - 1) / n_split;
    const int t0 = blockIdx.y * chunk;
    const int t1 = min(T, t0 + chunk);
    float* pout = partial + ((size_t)rh * n_split + blockIdx.y) * (D + 2);
    if (t0 >= t1) {
        write_empty_partial<D>(pout);
        return;
    }
    for (int d = threadIdx.x; d < D / 8; d += blockDim.x)
        *reinterpret_cast<uint4*>(s_q_sh + d * 8) = *reinterpret_cast<const uint4*>(q + (size_t)r * ldq + h * D + d * 8);
    __syncthreads();
    attend_chunk<D>(s_q_sh, CacheRows{L, b, h}, t0, t1, scale, pout, false, [] { return (bf16*)nullptr; });
}

// Fused single-token attention step: RoPE on the new q and k (rope.cuh, as rope_kernel), append
// k / v to the paged cache (hf cache_utils.py:119-120) and attend over positions 0 .. pos -- one launch instead of
// rope + kv_append + attention (+ combine when n_split == 1).  qkv: [batch, 3*H] pre-RoPE rows of the new token.
// RAGGED: row b's new token is at pos0 (+ *pos_dev) + row_off[b].
template <int D, bool RAGGED>
__global__ void __launch_bounds__(128)
decode_attn_fused_kernel(const bf16* __restrict__ qkv, KVLayout L, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                         float* __restrict__ partial, bf16* __restrict__ out, int pos0, const int* pos_dev, int ldq, int ldo,
                         float scale, int n_split, const int* __restrict__ row_off) {
    __shared__ __align__(16) bf16 s_q[D];
    __shared__ __align__(16) bf16 s_k[D];
    __shared__ __align__(16) bf16 s_v[D];
    const int rh = blockIdx.x;
    const int b = rh / L.n_heads, h = rh % L.n_heads;
    int pos = (pos_dev ? *pos_dev : 0) + pos0;           // position of the new token
    if constexpr (RAGGED) pos += row_off[b];
    const int T = pos + 1;
    const int chunk = (T + n_split - 1) / n_split;
    const int t0 = blockIdx.y * chunk;
    const int t1 = min(T, t0 + chunk);
    const int H = L.n_heads * D;
    const bf16* row = qkv + (size_t)b * ldq;
    const bool owns_new = (t0 <= pos && pos < t1);
    // RoPE(q) -> s_q ; the CTA whose chunk holds the new position also forms RoPE(k), v and appends them to the cache
    for (int i = threadIdx.x; i < D / 2; i += blockDim.x) {
        const float c = __bfloat162float(cos_t[(size_t)pos * (D / 2) + i]), sn = __bfloat162float(sin_t[(size_t)pos * (D / 2) + i]);
        {
            const float x1 = __bfloat162float(row[h * D + i]), x2 = __bfloat162float(row[h * D + i + D / 2]);
            s_q[i] = __float2bfloat16_rn(rope_fwd_elem(x1, x2, c, sn, false));
            s_q[i + D / 2] = __float2bfloat16_rn(rope_fwd_elem(x2, x1, c, sn, true));
        }
        if (owns_new) {
            const float x1 = __bfloat162float(row[H + h * D + i]), x2 = __bfloat162float(row[H + h * D + i + D / 2]);
            s_k[i] = __float2bfloat16_rn(rope_fwd_elem(x1, x2, c, sn, false));
            s_k[i + D / 2] = __float2bfloat16_rn(rope_fwd_elem(x2, x1, c, sn, true));
            s_v[i] = row[2 * H + h * D + i];
            s_v[i + D / 2] = row[2 * H + h * D + i + D / 2];
        }
    }
    __syncthreads();
    if (owns_new) {
        const size_t o = kv_off(L, b, h, pos);
        for (int i = threadIdx.x; i < D / 8; i += blockDim.x) {
            *reinterpret_cast<uint4*>(L.k_pool + o + i * 8) = *reinterpret_cast<const uint4*>(s_k + i * 8);
            *reinterpret_cast<uint4*>(L.v_pool + o + i * 8) = *reinterpret_cast<const uint4*>(s_v + i * 8);
        }
    }
    float* pout = partial + ((size_t)rh * n_split + blockIdx.y) * (D + 2);
    if (t0 >= t1) {
        write_empty_partial<D>(pout);
        return;
    }
    // n_split == 1: the whole context is in this CTA, which normalises and writes the attention output directly
    attend_chunk<D>(s_q, CacheRowsWithNew{{L, b, h}, s_k, s_v, pos}, t0, t1, scale, pout, n_split == 1,
                    [&] { return out + (size_t)b * ldo + h * D; });
}

// Token-level stack variant (context <= 32 positions): one WARP per (batch row, head); each lane owns D/32 consecutive
// elements of q / k / v, scores are warp reductions, softmax lives in registers.  Same math and rounding points as
// decode_attn_fused_kernel (RoPE three roundings, P rounded to bf16 before P.V).
template <int D, bool RAGGED>
__global__ void __launch_bounds__(128)
decode_attn_small_kernel(const bf16* __restrict__ qkv, KVLayout L, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                         bf16* __restrict__ out, int n_rows_heads, int pos0, const int* pos_dev, int ldq, int ldo, float scale,
                         const int* __restrict__ row_off) {
    constexpr int E = D / 32;          // elements per lane (8 for D = 256)
    static_assert(E == 8, "one 16-byte vector per lane");
    const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (wid >= n_rows_heads) return;
    const int lane = threadIdx.x & 31;
    const int b = wid / L.n_heads, h = wid % L.n_heads;
    int pos = (pos_dev ? *pos_dev : 0) + pos0;
    if constexpr (RAGGED) pos += row_off[b];
    const int H = L.n_heads * D;
    const bf16* row = qkv + (size_t)b * ldq + h * D;
    // RoPE pairs (d, d + D/2) live in lanes l and l ^ 16.  q and k are rotated in one loop rather than by two calls of
    // rope_fwd_lane: the compiler schedules the shuffles of both together
    float qv[8], kv_[8], cs[8], sn[8];
    unpack8(*reinterpret_cast<const uint4*>(row + lane * 8), qv);
    unpack8(*reinterpret_cast<const uint4*>(row + H + lane * 8), kv_);
    unpack8(*reinterpret_cast<const uint4*>(cos_t + (size_t)pos * (D / 2) + (lane & 15) * 8), cs);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + (size_t)pos * (D / 2) + (lane & 15) * 8), sn);
    float qr[8], kr[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const float qo = __shfl_xor_sync(0xffffffffu, qv[j], 16), ko = __shfl_xor_sync(0xffffffffu, kv_[j], 16);
        qr[j] = bf16_round(rope_fwd_elem(qv[j], qo, cs[j], sn[j], lane >= 16));
        kr[j] = bf16_round(rope_fwd_elem(kv_[j], ko, cs[j], sn[j], lane >= 16));
    }
    const uint4 k_new = pack8(kr);
    const uint4 v_new = *reinterpret_cast<const uint4*>(row + 2 * H + lane * 8);
    {
        const size_t o = kv_off(L, b, h, pos) + lane * 8;
        *reinterpret_cast<uint4*>(L.k_pool + o) = k_new;
        *reinterpret_cast<uint4*>(L.v_pool + o) = v_new;
    }
    const int T = pos + 1;             // <= 32
    float my_s = -INFINITY;            // lane t keeps the score of key t
    for (int t = 0; t < T; t++) {
        float kf[8];
        if (t == pos) unpack8(k_new, kf);
        else unpack8(*reinterpret_cast<const uint4*>(L.k_pool + kv_off(L, b, h, t) + lane * 8), kf);
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; j++) s = fmaf(kf[j], qr[j], s);
        s = warp_sum(s) * scale;
        if (lane == t) my_s = s;
    }
    const float mx = warp_max(my_s);
    const float p = (lane < T) ? __expf(my_s - mx) : 0.f;
    const float sum = warp_sum(p);
    const float pb = bf16_round(p);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int t = 0; t < T; t++) {
        const float pt = __shfl_sync(0xffffffffu, pb, t);
        float vf[8];
        if (t == pos) unpack8(v_new, vf);
        else unpack8(*reinterpret_cast<const uint4*>(L.v_pool + kv_off(L, b, h, t) + lane * 8), vf);
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = fmaf(pt, vf[j], acc[j]);
    }
    const float inv = 1.f / sum;
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] *= inv;
    *reinterpret_cast<uint4*>(out + (size_t)b * ldo + h * D + lane * 8) = pack8(acc);
}

template <int D>
__global__ void decode_attn_combine_kernel(const float* __restrict__ partial, bf16* __restrict__ out, int n_heads,
                                           int n_split, int ldo) {
    const int rh = blockIdx.x;
    const int r = rh / n_heads, h = rh % n_heads;
    const float* p = partial + (size_t)rh * n_split * (D + 2);
    float mx = -INFINITY;
    for (int s = 0; s < n_split; s++) mx = fmaxf(mx, p[s * (D + 2)]);
    float l = 0.f;
    for (int s = 0; s < n_split; s++) {
        const float m = p[s * (D + 2)];
        if (m > -INFINITY) l += p[s * (D + 2) + 1] * __expf(m - mx);
    }
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float o = 0.f;
        for (int s = 0; s < n_split; s++) {
            const float m = p[s * (D + 2)];
            if (m > -INFINITY) o += p[s * (D + 2) + 2 + d] * __expf(m - mx);
        }
        out[(size_t)r * ldo + h * D + d] = __float2bfloat16_rn(o / l);
    }
}

// ---------------------------------------------------------------------------------------------
// sampler (helpers in sampler.cuh, shared with the persistent decode kernel)
// ---------------------------------------------------------------------------------------------
constexpr int SMP_THREADS = 256;
constexpr int SMP_MAXV = smp::SMP_MAXV;
using smp::key_before;

// probs: [rows, V] (bf16 or fp32) already softmaxed and masked (public sample_top_p_k API)
template <typename T>
__global__ void __launch_bounds__(SMP_THREADS)
sample_probs_kernel(const T* __restrict__ probs, int V, int ld, float top_p, int top_k, const float* __restrict__ uniforms,
                    long long* __restrict__ out, bool bf16_sem) {
    __shared__ float s_p[SMP_MAXV];
    __shared__ int s_i[SMP_MAXV];
    __shared__ int s_cnt[SMP_THREADS + 1];
    const int r = blockIdx.x;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        float p = (float)probs[(size_t)r * ld + i];
        s_p[i] = (p > 0.f) ? p : 0.f;   // NaN / negative -> 0
    }
    __syncthreads();
    const int n = smp::compact_nonzero<SMP_THREADS>(s_p, s_i, V, s_cnt);
    const int id = smp::sample_tail<SMP_THREADS>(s_p, s_i, n, top_p, top_k, uniforms[r], bf16_sem);
    if (threadIdx.x == 0) out[r] = id;
}

// Fused generate-step sampler: logits [rows, ld] bf16 -> token id.
// Allowed ids of row r at inner step `step` (midi_model.py:202-215):
//   step 0            : [eos_id, eos_id + n_event_types]  (eos + the event-type ids, contiguous)
//   step i > 0        : lut[(ev - first_event) * 8 + (i-1)] = (lo, hi) of that parameter; pad only if exhausted / ended
// `event_tok` [rows] holds the step-0 token of the current event; `dense_mask` (optional, [rows, V] uint8) is ANDed.
// ROWS: row r samples with row_temp[r], row_top_p[r], row_top_k[r] instead of the scalar settings.
template <bool ROWS>
__global__ void __launch_bounds__(SMP_THREADS)
sample_logits_kernel(const bf16* __restrict__ logits, int V, int ld, float temp, float top_p, int top_k, int step,
                     const long long* __restrict__ event_tok, const int* __restrict__ lut, int n_event_types, int eos_id,
                     int pad_id, const unsigned char* __restrict__ dense_mask, const float* __restrict__ uniforms,
                     long long* __restrict__ out, int out_stride, const float* __restrict__ row_temp,
                     const float* __restrict__ row_top_p, const int* __restrict__ row_top_k) {
    __shared__ float s_p[SMP_MAXV];
    __shared__ int s_i[SMP_MAXV];
    __shared__ int s_cnt[SMP_THREADS + 8];
    __shared__ float s_red[64];
    const int r = blockIdx.x;
    if constexpr (ROWS) {
        temp = row_temp[r];
        top_p = row_top_p[r];
        top_k = row_top_k[r];
    }
    int lo, hi;
    if (step == 0) {
        lo = eos_id; hi = eos_id + 1 + n_event_types;
    } else {
        const long long ev = event_tok[r];
        const int e = (int)ev - (eos_id + 1);
        if (ev == eos_id || e < 0 || e >= n_event_types) { lo = pad_id; hi = pad_id + 1; }
        else {
            lo = lut[(e * 8 + (step - 1)) * 2];
            hi = lut[(e * 8 + (step - 1)) * 2 + 1];
            if (hi <= lo) { lo = pad_id; hi = pad_id + 1; }
        }
    }
    // temperature softmax, grammar range / mask, top-p, top-k, draw (sampler.cuh)
    const int id = smp::sample_logits_row<SMP_THREADS>(logits + (size_t)r * ld, V, temp, top_p, top_k, lo, hi,
                                                       dense_mask ? dense_mask + (size_t)r * V : nullptr, uniforms[r], s_p, s_i,
                                                       s_cnt, s_red, false);
    if (threadIdx.x == 0) out[(size_t)r * out_stride] = id;
}

// counter-based uniform generator for graph-captured loops: u[r] = hash(seed ^ state[1], state[0], r) in [0,1);
// state = {call counter, device-side seed} so that a captured graph can be re-seeded without re-capture
__global__ void philox_uniform_kernel(float* __restrict__ u, int n, unsigned long long seed, unsigned long long* counter) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long c = counter[0];
    seed ^= counter[1];
    if (i < n) u[i] = smp::counter_uniform(seed, c, (unsigned long long)i);
    __syncthreads();
    if (i == 0) *counter = c + 1;
}

// Keyed uniforms of the per-request queue: row b's draw at token step `step` of its new event j = *pos + row_off[b] -
// row_first[b] is the draw of generating the request alone (batch 1, row 0, seed row_seed[b]): hash(row_seed[b], 8 j + step,
// 0).  The position is read on the device, so a captured graph replays it.
__global__ void uniform_rows_kernel(float* __restrict__ u, int B, const int* __restrict__ pos, const int* __restrict__ row_off,
                                    const int* __restrict__ row_first, const unsigned long long* __restrict__ row_seed,
                                    int step) {
    const int b = threadIdx.x;
    if (b < B) {
        const int j = *pos + row_off[b] - row_first[b];
        u[b] = smp::counter_uniform(row_seed[b], (unsigned long long)j * 8ULL + (unsigned long long)step, 0ULL);
    }
}

// End of one generated event (graph-captured loop): ev_t [T][B] (token-major scratch written by the sampler)
// -> seq[b, *pos + 1, :] (RAGGED: seq[b, *pos + row_off[b] + 1, :]) and ev_next[b, :] (input of the next outer step);
// then (*pos)++.
template <bool RAGGED>
__global__ void event_commit_kernel(const long long* __restrict__ ev_t, long long* __restrict__ seq,
                                    long long* __restrict__ ev_next, int* __restrict__ pos, int B, int T, int max_len,
                                    const int* __restrict__ row_off) {
    const int p = *pos;
    for (int i = threadIdx.x; i < B * T; i += blockDim.x) {
        const int b = i / T, t = i % T;
        const long long v = ev_t[(size_t)t * B + b];
        int q = p;
        if constexpr (RAGGED) q += row_off[b];
        if (q + 1 < max_len) seq[((size_t)b * max_len + q + 1) * T + t] = v;
        ev_next[(size_t)b * T + t] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) *pos = p + 1;
}

// event_commit_kernel<true> of the request-queue loop, with the persistent queue kernel's per-row finish rule: only a live
// row (row_last[b] == -1) commits, and it finishes when its committed event is EOS or lands on row_end[b], its seq index
// then going to row_last[b].
__global__ void event_commit_queue_kernel(const long long* __restrict__ ev_t, long long* __restrict__ seq,
                                          long long* __restrict__ ev_next, int* __restrict__ pos, int B, int T, int max_len,
                                          const int* __restrict__ row_off, const int* __restrict__ row_end,
                                          int* __restrict__ row_last, int eos_id) {
    const int p = *pos;
    for (int i = threadIdx.x; i < B * T; i += blockDim.x) {
        const int b = i / T, t = i % T;
        if (row_last[b] != -1) continue;
        const long long v = ev_t[(size_t)t * B + b];
        const int q = p + row_off[b];
        if (q + 1 < max_len) seq[((size_t)b * max_len + q + 1) * T + t] = v;
        ev_next[(size_t)b * T + t] = v;
    }
    __syncthreads();                                     // every read of row_last above precedes its writes below
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        if (row_last[b] != -1) continue;
        const int last = p + row_off[b] + 1;
        if (ev_t[b] == eos_id || last >= row_end[b]) row_last[b] = last;
    }
    if (threadIdx.x == 0) *pos = p + 1;
}

}   // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" int b200_gemv_bf16(const void* x, const void* W, const void* res, void* y, int B, int N, int K, int ldx, int ldw,
                              int ldr, int ldy, cudaStream_t stream) {
    B200_CHECK_ARG(B >= 1 && B <= 16, "gemv: batch %d outside 1..16 (use the tensor-core GEMM)", B);
    B200_CHECK_ARG(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "gemv: K, ldx, ldw must be multiples of 8");
    const size_t smem = (size_t)B * K * 2;
    B200_CHECK_ARG(smem <= 200 * 1024, "gemv: B*K too large for shared memory");
    int grid = (N + GV_WARPS - 1) / GV_WARPS;
    const int cap = b200_num_sms() * 4;
    if (grid > cap) grid = cap;
#define B200_GEMV(BB)                                                                                              \
    do {                                                                                                           \
        static bool configured = false;                                                                            \
        if (!configured) {                                                                                         \
            B200_CUDA(cudaFuncSetAttribute(gemv_kernel<BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024), \
                      "gemv smem attr");                                                                           \
            configured = true;                                                                                     \
        }                                                                                                          \
        gemv_kernel<BB><<<grid, GV_WARPS * 32, smem, stream>>>((const bf16*)x, (const bf16*)W, (const bf16*)res,   \
                                                               (bf16*)y, N, K, ldx, ldw, ldr, ldy);                \
    } while (0)
    switch (B) {
        case 1: B200_GEMV(1); break;
        case 2: B200_GEMV(2); break;
        case 3: B200_GEMV(3); break;
        case 4: B200_GEMV(4); break;
        case 5: B200_GEMV(5); break;
        case 6: B200_GEMV(6); break;
        case 7: B200_GEMV(7); break;
        case 8: B200_GEMV(8); break;
        case 9: B200_GEMV(9); break;
        case 10: B200_GEMV(10); break;
        case 11: B200_GEMV(11); break;
        case 12: B200_GEMV(12); break;
        case 13: B200_GEMV(13); break;
        case 14: B200_GEMV(14); break;
        case 15: B200_GEMV(15); break;
        default: B200_GEMV(16); break;
    }
#undef B200_GEMV
    B200_CHECK_LAUNCH("gemv");
    return B200_OK;
}

extern "C" size_t b200_attn_decode_workspace_bytes(int rows, int n_heads, int head_dim, int n_split);

extern "C" int b200_gemv_fused(const void* x, const long long* ids, int ids_stride, const void* table, int V,
                               const void* norm_w, float eps, const void* W, const void* res, void* y, int B, int N_out, int K,
                               int ldx, int ldw, int ldr, int ldy, int swiglu, cudaStream_t stream) {
    B200_CHECK_ARG(B >= 1 && B <= 16, "gemv_fused: batch %d outside 1..16", B);
    B200_CHECK_ARG(K % 8 == 0 && ldw % 8 == 0 && (ids || ldx % 8 == 0), "gemv_fused: K, ldx, ldw must be multiples of 8");
    B200_CHECK_ARG(x != nullptr || ids != nullptr, "gemv_fused: x or ids required");
    const size_t smem = (size_t)B * K * 2;
    B200_CHECK_ARG(smem <= 200 * 1024, "gemv_fused: B*K too large for shared memory");
    int grid = (N_out + GV_WARPS - 1) / GV_WARPS;
    const int cap = b200_num_sms() * 4;
    if (grid > cap) grid = cap;
#define B200_GEMVF(BB)                                                                                                  \
    do {                                                                                                                \
        static bool configured = false;                                                                                 \
        if (!configured) {                                                                                              \
            B200_CUDA(cudaFuncSetAttribute(gemv_fused_kernel<BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024), \
                      "gemv_fused smem attr");                                                                          \
            configured = true;                                                                                          \
        }                                                                                                               \
        gemv_fused_kernel<BB><<<grid, GV_WARPS * 32, smem, stream>>>((const bf16*)x, ids, ids_stride, (const bf16*)table, \
            (const bf16*)norm_w, eps, (const bf16*)W, (const bf16*)res, (bf16*)y, N_out, K, ldx, ldw, ldr, ldy, swiglu, V); \
    } while (0)
    switch (B) {
        case 1: B200_GEMVF(1); break;
        case 2: B200_GEMVF(2); break;
        case 3: B200_GEMVF(3); break;
        case 4: B200_GEMVF(4); break;
        case 5: B200_GEMVF(5); break;
        case 6: B200_GEMVF(6); break;
        case 7: B200_GEMVF(7); break;
        case 8: B200_GEMVF(8); break;
        case 9: B200_GEMVF(9); break;
        case 10: B200_GEMVF(10); break;
        case 11: B200_GEMVF(11); break;
        case 12: B200_GEMVF(12); break;
        case 13: B200_GEMVF(13); break;
        case 14: B200_GEMVF(14); break;
        case 15: B200_GEMVF(15); break;
        default: B200_GEMVF(16); break;
    }
#undef B200_GEMVF
    B200_CHECK_LAUNCH("gemv_fused");
    return B200_OK;
}

namespace {

template <bool RAGGED>
int attn_decode_fused(const void* qkv, void* k_pool, void* v_pool, const int* block_table, int max_pages, int page,
                      const void* cos_t, const void* sin_t, void* out, int batch, int n_heads, int head_dim, int pos0,
                      const int* pos_dev, int max_T, int ldq, int ldo, float scale, int n_split, void* workspace,
                      size_t workspace_bytes, const int* row_off, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == 64 || head_dim == 256, "attn_decode_fused: head_dim %d unsupported", head_dim);
    if (batch == 0) return B200_OK;
    B200_CHECK_ARG(!RAGGED || row_off, "attn_decode_fused_ragged: row_off required");
    if (n_split < 1) n_split = 1;
    B200_CHECK_ARG((max_T + n_split - 1) / n_split <= 1024, "attn_decode_fused: chunk per split exceeds 1024 keys");
    B200_CHECK_ARG(workspace_bytes >= b200_attn_decode_workspace_bytes(batch, n_heads, head_dim, n_split),
                   "attn_decode_fused: workspace too small");
    KVLayout L{(bf16*)k_pool, (bf16*)v_pool, block_table, max_pages, page, n_heads, head_dim};
    if (head_dim == 256 && max_T <= 32) {      // token-level stack: warp-per-head kernel
        const int n = batch * n_heads;
        decode_attn_small_kernel<256, RAGGED><<<(n + 3) / 4, 128, 0, stream>>>((const bf16*)qkv, L, (const bf16*)cos_t,
            (const bf16*)sin_t, (bf16*)out, n, pos0, pos_dev, ldq, ldo, scale, row_off);
        B200_CHECK_LAUNCH("attn_decode_small");
        return B200_OK;
    }
    dim3 grid(batch * n_heads, n_split);
    if (head_dim == 64) {
        decode_attn_fused_kernel<64, RAGGED><<<grid, 128, 0, stream>>>((const bf16*)qkv, L, (const bf16*)cos_t, (const bf16*)sin_t,
            (float*)workspace, (bf16*)out, pos0, pos_dev, ldq, ldo, scale, n_split, row_off);
        if (n_split > 1) {
            decode_attn_combine_kernel<64><<<batch * n_heads, 64, 0, stream>>>((const float*)workspace, (bf16*)out, n_heads, n_split, ldo);
            B200_COUNT_EXTRA(1);
        }
    } else {
        decode_attn_fused_kernel<256, RAGGED><<<grid, 128, 0, stream>>>((const bf16*)qkv, L, (const bf16*)cos_t, (const bf16*)sin_t,
            (float*)workspace, (bf16*)out, pos0, pos_dev, ldq, ldo, scale, n_split, row_off);
        if (n_split > 1) {
            decode_attn_combine_kernel<256><<<batch * n_heads, 128, 0, stream>>>((const float*)workspace, (bf16*)out, n_heads, n_split, ldo);
            B200_COUNT_EXTRA(1);
        }
    }
    B200_CHECK_LAUNCH("attn_decode_fused");
    return B200_OK;
}

template <bool RAGGED>
int kv_append(const void* qkv, void* k_pool, void* v_pool, const int* block_table, int max_pages, int page, int n_heads,
              int head_dim, int batch, int s_new, int pos0, const int* pos0_dev, int ld, const int* row_off,
              cudaStream_t stream) {
    B200_CHECK_ARG(head_dim % 8 == 0, "kv_append: head_dim must be a multiple of 8");
    if (batch * s_new == 0) return B200_OK;
    B200_CHECK_ARG(!RAGGED || row_off, "kv_append_ragged: row_off required");
    KVLayout L{(bf16*)k_pool, (bf16*)v_pool, block_table, max_pages, page, n_heads, head_dim};
    kv_append_kernel<RAGGED><<<batch * s_new, 128, 0, stream>>>((const bf16*)qkv, L, s_new, pos0, pos0_dev, ld, row_off);
    B200_CHECK_LAUNCH("kv_append");
    return B200_OK;
}

template <bool RAGGED>
int attn_decode(const void* q, const void* k_pool, const void* v_pool, const int* block_table, int max_pages, int page,
                void* out, int batch, int s_q, int n_heads, int head_dim, int past, const int* past_dev, int max_T, int ldq,
                int ldo, float scale, int n_split, void* workspace, size_t workspace_bytes, const int* row_off,
                cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == 64 || head_dim == 256, "attn_decode: head_dim %d unsupported", head_dim);
    const int rows = batch * s_q;
    if (rows == 0) return B200_OK;
    B200_CHECK_ARG(!RAGGED || row_off, "attn_decode_ragged: row_off required");
    if (n_split < 1) n_split = 1;
    B200_CHECK_ARG((max_T + n_split - 1) / n_split <= 1024, "attn_decode: chunk per split exceeds 1024 keys (raise n_split)");
    B200_CHECK_ARG(workspace_bytes >= b200_attn_decode_workspace_bytes(rows, n_heads, head_dim, n_split),
                   "attn_decode: workspace too small");
    KVLayout L{(bf16*)k_pool, (bf16*)v_pool, block_table, max_pages, page, n_heads, head_dim};
    dim3 grid(rows * n_heads, n_split);
    if (head_dim == 64) {
        decode_attn_kernel<64, RAGGED><<<grid, 128, 0, stream>>>((const bf16*)q, L, (float*)workspace, s_q, past, past_dev, ldq,
                                                                 scale, n_split, row_off);
        decode_attn_combine_kernel<64><<<rows * n_heads, 64, 0, stream>>>((const float*)workspace, (bf16*)out, n_heads, n_split, ldo);
    } else {
        decode_attn_kernel<256, RAGGED><<<grid, 128, 0, stream>>>((const bf16*)q, L, (float*)workspace, s_q, past, past_dev, ldq,
                                                                  scale, n_split, row_off);
        decode_attn_combine_kernel<256><<<rows * n_heads, 128, 0, stream>>>((const float*)workspace, (bf16*)out, n_heads, n_split, ldo);
    }
    B200_COUNT_EXTRA(1);
    B200_CHECK_LAUNCH("attn_decode");
    return B200_OK;
}

}   // namespace

// one new token per batch row: RoPE(q,k) + KV append + attention over the cache (+ combine pass when n_split > 1)
extern "C" int b200_attn_decode_fused(const void* qkv, void* k_pool, void* v_pool, const int* block_table, int max_pages,
                                      int page, const void* cos_t, const void* sin_t, void* out, int batch, int n_heads,
                                      int head_dim, int pos0, const int* pos_dev, int max_T, int ldq, int ldo, float scale,
                                      int n_split, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    return attn_decode_fused<false>(qkv, k_pool, v_pool, block_table, max_pages, page, cos_t, sin_t, out, batch, n_heads,
                                    head_dim, pos0, pos_dev, max_T, ldq, ldo, scale, n_split, workspace, workspace_bytes,
                                    nullptr, stream);
}

extern "C" int b200_attn_decode_fused_ragged(const void* qkv, void* k_pool, void* v_pool, const int* block_table,
                                             int max_pages, int page, const void* cos_t, const void* sin_t, void* out,
                                             int batch, int n_heads, int head_dim, int pos0, const int* pos_dev, int max_T,
                                             int ldq, int ldo, float scale, int n_split, void* workspace,
                                             size_t workspace_bytes, const int* row_off, cudaStream_t stream) {
    return attn_decode_fused<true>(qkv, k_pool, v_pool, block_table, max_pages, page, cos_t, sin_t, out, batch, n_heads,
                                   head_dim, pos0, pos_dev, max_T, ldq, ldo, scale, n_split, workspace, workspace_bytes,
                                   row_off, stream);
}

extern "C" int b200_kv_append(const void* qkv, void* k_pool, void* v_pool, const int* block_table, int max_pages, int page,
                              int n_heads, int head_dim, int batch, int s_new, int pos0, const int* pos0_dev, int ld,
                              cudaStream_t stream) {
    return kv_append<false>(qkv, k_pool, v_pool, block_table, max_pages, page, n_heads, head_dim, batch, s_new, pos0,
                            pos0_dev, ld, nullptr, stream);
}

extern "C" int b200_kv_append_ragged(const void* qkv, void* k_pool, void* v_pool, const int* block_table, int max_pages,
                                     int page, int n_heads, int head_dim, int batch, int s_new, int pos0,
                                     const int* pos0_dev, int ld, const int* row_off, cudaStream_t stream) {
    return kv_append<true>(qkv, k_pool, v_pool, block_table, max_pages, page, n_heads, head_dim, batch, s_new, pos0,
                           pos0_dev, ld, row_off, stream);
}

extern "C" size_t b200_attn_decode_workspace_bytes(int rows, int n_heads, int head_dim, int n_split) {
    return (size_t)rows * n_heads * n_split * (head_dim + 2) * sizeof(float);
}

// q: [batch*s_q, ldq] (q third of the packed qkv row, post-RoPE); out: [batch*s_q, ldo]
extern "C" int b200_attn_decode(const void* q, const void* k_pool, const void* v_pool, const int* block_table, int max_pages,
                                int page, void* out, int batch, int s_q, int n_heads, int head_dim, int past,
                                const int* past_dev, int max_T, int ldq, int ldo, float scale, int n_split, void* workspace,
                                size_t workspace_bytes, cudaStream_t stream) {
    return attn_decode<false>(q, k_pool, v_pool, block_table, max_pages, page, out, batch, s_q, n_heads, head_dim, past,
                              past_dev, max_T, ldq, ldo, scale, n_split, workspace, workspace_bytes, nullptr, stream);
}

extern "C" int b200_attn_decode_ragged(const void* q, const void* k_pool, const void* v_pool, const int* block_table,
                                       int max_pages, int page, void* out, int batch, int s_q, int n_heads, int head_dim,
                                       int past, const int* past_dev, int max_T, int ldq, int ldo, float scale, int n_split,
                                       void* workspace, size_t workspace_bytes, const int* row_off, cudaStream_t stream) {
    return attn_decode<true>(q, k_pool, v_pool, block_table, max_pages, page, out, batch, s_q, n_heads, head_dim, past,
                             past_dev, max_T, ldq, ldo, scale, n_split, workspace, workspace_bytes, row_off, stream);
}

extern "C" int b200_sample_topp_topk(const void* probs, int is_bf16, int rows, int V, int ld, float top_p, int top_k,
                                     const float* uniforms, long long* out, cudaStream_t stream) {
    B200_CHECK_ARG(V <= SMP_MAXV, "sample_topp_topk: vocabulary %d exceeds %d", V, SMP_MAXV);
    if (rows == 0) return B200_OK;
    if (top_k < 1) top_k = 1;
    if (is_bf16)
        sample_probs_kernel<bf16><<<rows, SMP_THREADS, 0, stream>>>((const bf16*)probs, V, ld, top_p, top_k, uniforms, out, true);
    else
        sample_probs_kernel<float><<<rows, SMP_THREADS, 0, stream>>>((const float*)probs, V, ld, top_p, top_k, uniforms, out, false);
    B200_CHECK_LAUNCH("sample_topp_topk");
    return B200_OK;
}

extern "C" int b200_sample_from_logits(const void* logits, int rows, int V, int ld, float temp, float top_p, int top_k,
                                       int step, const long long* event_tok, const int* lut, int n_event_types, int eos_id,
                                       int pad_id, const unsigned char* dense_mask, const float* uniforms, long long* out,
                                       int out_stride, cudaStream_t stream) {
    B200_CHECK_ARG(V <= SMP_MAXV, "sample_from_logits: vocabulary %d exceeds %d", V, SMP_MAXV);
    B200_CHECK_ARG(temp > 0.f, "sample_from_logits: temperature must be positive");
    if (rows == 0) return B200_OK;
    if (top_k < 1) top_k = 1;
    sample_logits_kernel<false><<<rows, SMP_THREADS, 0, stream>>>((const bf16*)logits, V, ld, temp, top_p, top_k, step,
                                                                 event_tok, lut, n_event_types, eos_id, pad_id, dense_mask,
                                                                 uniforms, out, out_stride, nullptr, nullptr, nullptr);
    B200_CHECK_LAUNCH("sample_from_logits");
    return B200_OK;
}

extern "C" int b200_sample_from_logits_rows(const void* logits, int rows, int V, int ld, const float* row_temp,
                                            const float* row_top_p, const int* row_top_k, int step, const long long* event_tok,
                                            const int* lut, int n_event_types, int eos_id, int pad_id,
                                            const unsigned char* dense_mask, const float* uniforms, long long* out,
                                            int out_stride, cudaStream_t stream) {
    B200_CHECK_ARG(V <= SMP_MAXV, "sample_from_logits_rows: vocabulary %d exceeds %d", V, SMP_MAXV);
    B200_CHECK_ARG(row_temp != nullptr && row_top_p != nullptr && row_top_k != nullptr,
                   "sample_from_logits_rows: row_temp, row_top_p and row_top_k required");
    if (rows == 0) return B200_OK;
    sample_logits_kernel<true><<<rows, SMP_THREADS, 0, stream>>>((const bf16*)logits, V, ld, 1.f, 1.f, 1, step, event_tok,
                                                                lut, n_event_types, eos_id, pad_id, dense_mask, uniforms,
                                                                out, out_stride, row_temp, row_top_p, row_top_k);
    B200_CHECK_LAUNCH("sample_from_logits_rows");
    return B200_OK;
}

extern "C" int b200_uniform_fill(float* u, int n, unsigned long long seed, unsigned long long* counter_dev,
                                 cudaStream_t stream) {
    B200_CHECK_ARG(n >= 1 && n <= 1024, "uniform_fill: n outside 1..1024");
    philox_uniform_kernel<<<1, 1024, 0, stream>>>(u, n, seed, counter_dev);
    B200_CHECK_LAUNCH("uniform_fill");
    return B200_OK;
}

extern "C" int b200_uniform_fill_rows(float* u, int B, const int* pos_dev, const int* row_off, const int* row_first,
                                      const unsigned long long* row_seed, int step, cudaStream_t stream) {
    B200_CHECK_ARG(B >= 1 && B <= 1024, "uniform_fill_rows: B outside 1..1024");
    B200_CHECK_ARG(pos_dev != nullptr && row_off != nullptr && row_first != nullptr && row_seed != nullptr,
                   "uniform_fill_rows: pos, row_off, row_first and row_seed required");
    uniform_rows_kernel<<<1, (B + 31) / 32 * 32, 0, stream>>>(u, B, pos_dev, row_off, row_first, row_seed, step);
    B200_CHECK_LAUNCH("uniform_fill_rows");
    return B200_OK;
}

extern "C" int b200_event_commit(const long long* ev_t, long long* seq, long long* ev_next, int* pos_dev, int B, int T,
                                 int max_len, cudaStream_t stream) {
    event_commit_kernel<false><<<1, 256, 0, stream>>>(ev_t, seq, ev_next, pos_dev, B, T, max_len, nullptr);
    B200_CHECK_LAUNCH("event_commit");
    return B200_OK;
}

extern "C" int b200_event_commit_ragged(const long long* ev_t, long long* seq, long long* ev_next, int* pos_dev, int B,
                                        int T, int max_len, const int* row_off, cudaStream_t stream) {
    B200_CHECK_ARG(row_off != nullptr, "event_commit_ragged: row_off required");
    event_commit_kernel<true><<<1, 256, 0, stream>>>(ev_t, seq, ev_next, pos_dev, B, T, max_len, row_off);
    B200_CHECK_LAUNCH("event_commit");
    return B200_OK;
}

extern "C" int b200_event_commit_queue(const long long* ev_t, long long* seq, long long* ev_next, int* pos_dev, int B, int T,
                                       int max_len, const int* row_off, const int* row_end, int* row_last, int eos_id,
                                       cudaStream_t stream) {
    B200_CHECK_ARG(row_off != nullptr && row_end != nullptr && row_last != nullptr,
                   "event_commit_queue: row_off, row_end and row_last required");
    event_commit_queue_kernel<<<1, 256, 0, stream>>>(ev_t, seq, ev_next, pos_dev, B, T, max_len, row_off, row_end, row_last,
                                                     eos_id);
    B200_CHECK_LAUNCH("event_commit_queue");
    return B200_OK;
}
