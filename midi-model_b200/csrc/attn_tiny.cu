// Attention of the inner token stack: every event is an independent causal problem of
// L <= 8 positions with head_dim 256 (midi_model.py:116-135 -> hf sdpa, scale 1/16).  A flash
// tile would be >= 94 % padding, so one warp owns one (event, head): each lane holds an
// 8-wide slice of d for all L rows in registers, the L(L+1)/2 scores are reduced with warp
// shuffles, softmax is fp32, P is rounded to bf16 before P.V (flash semantics, DESIGN.md 3.3).
// HBM-bound: reads the packed qkv rows once, writes the output once.
#include "common.cuh"
#include "rope.cuh"

namespace {

constexpr int TD = 256;              // head_dim (32 lanes x 8)
constexpr int WARPS_PER_CTA = 4;

__device__ __forceinline__ float dot8(const uint4& a, const uint4& b) {
    const bf162* pa = reinterpret_cast<const bf162*>(&a);
    const bf162* pb = reinterpret_cast<const bf162*>(&b);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float2 x = __bfloat1622float2(pa[i]), y = __bfloat1622float2(pb[i]);
        s = fmaf(x.x, y.x, s);
        s = fmaf(x.y, y.y, s);
    }
    return s;
}
__device__ __forceinline__ void axpy8(float* acc, float a, const uint4& x) {
    const bf162* px = reinterpret_cast<const bf162*>(&x);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float2 v = __bfloat1622float2(px[i]);
        acc[2 * i] = fmaf(a, v.x, acc[2 * i]);
        acc[2 * i + 1] = fmaf(a, v.y, acc[2 * i + 1]);
    }
}

// RoPE backward / forward on the lane's slice of head_dim 256 at position pos (tables are [pos][128])
__device__ __forceinline__ void rope_bwd_slice(float* acc, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                               int pos, int lane) {
    float c[8], sn[8];
    unpack8(*reinterpret_cast<const uint4*>(cos_t + (size_t)pos * (TD / 2) + (lane & 15) * 8), c);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + (size_t)pos * (TD / 2) + (lane & 15) * 8), sn);
    rope_bwd_lane(acc, c, sn, lane);
}
__device__ __forceinline__ uint4 rope_fwd_slice(const uint4& x, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                                int pos, int lane) {
    float v[8], c[8], sn[8];
    unpack8(x, v);
    unpack8(*reinterpret_cast<const uint4*>(cos_t + (size_t)pos * (TD / 2) + (lane & 15) * 8), c);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + (size_t)pos * (TD / 2) + (lane & 15) * 8), sn);
    rope_fwd_lane(v, c, sn, lane);
    return pack8(v);
}

// causal softmax over s[i][0..i] (scaled scores); returns fp32 probabilities in place
template <int L>
__device__ __forceinline__ void softmax_rows(float s[L][L]) {
#pragma unroll
    for (int i = 0; i < L; i++) {
        float m = s[i][0];
#pragma unroll
        for (int j = 1; j <= i; j++) m = fmaxf(m, s[i][j]);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j <= i; j++) {
            s[i][j] = __expf(s[i][j] - m);
            sum += s[i][j];
        }
        const float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j <= i; j++) s[i][j] *= inv;
    }
}

template <int L>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
tiny_attn_fwd_kernel(bf16* __restrict__ qkv, bf16* __restrict__ out, int n_events, int n_heads, int ld_qkv, int ld_out,
                     float scale, const bf16* __restrict__ rope_cos, const bf16* __restrict__ rope_sin) {
    B200_PDL_TRIGGER();
    const int wid = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (wid >= n_events * n_heads) return;
    const int lane = threadIdx.x & 31;
    const int e = wid / n_heads, h = wid % n_heads;
    const int H = n_heads * TD;
    bf16* base = qkv + (size_t)e * L * ld_qkv + h * TD + lane * 8;
    uint4 q[L], k[L];
#pragma unroll
    for (int i = 0; i < L; i++) {
        q[i] = *reinterpret_cast<const uint4*>(base + (size_t)i * ld_qkv);
        k[i] = *reinterpret_cast<const uint4*>(base + (size_t)i * ld_qkv + H);
    }
    if (rope_cos) {
        // fused RoPE: this warp owns the (event, head) slice, so q and k are rotated in registers and written back in
        // place -- the saved activation is post-RoPE, as the backward pass expects
#pragma unroll
        for (int i = 0; i < L; i++) {
            q[i] = rope_fwd_slice(q[i], rope_cos, rope_sin, i, lane);
            k[i] = rope_fwd_slice(k[i], rope_cos, rope_sin, i, lane);
            *reinterpret_cast<uint4*>(base + (size_t)i * ld_qkv) = q[i];
            *reinterpret_cast<uint4*>(base + (size_t)i * ld_qkv + H) = k[i];
        }
    }
    float s[L][L];
#pragma unroll
    for (int i = 0; i < L; i++)
#pragma unroll
        for (int j = 0; j <= i; j++) s[i][j] = warp_sum(dot8(q[i], k[j])) * scale;
    softmax_rows<L>(s);
    uint4 v[L];
#pragma unroll
    for (int i = 0; i < L; i++) v[i] = ld_nc16(base + (size_t)i * ld_qkv + 2 * H);
#pragma unroll
    for (int i = 0; i < L; i++) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j <= i; j++) axpy8(acc, bf16_round(s[i][j]), v[j]);
        *reinterpret_cast<uint4*>(out + ((size_t)e * L + i) * ld_out + h * TD + lane * 8) = pack8(acc);
    }
}

template <int L>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
tiny_attn_bwd_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ d_out, bf16* __restrict__ dqkv, int n_events,
                     int n_heads, int ld_qkv, int ld_out, float scale, const bf16* __restrict__ rope_cos,
                     const bf16* __restrict__ rope_sin) {
    B200_PDL_TRIGGER();
    const int wid = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (wid >= n_events * n_heads) return;
    const int lane = threadIdx.x & 31;
    const int e = wid / n_heads, h = wid % n_heads;
    const int H = n_heads * TD;
    const size_t col = (size_t)h * TD + lane * 8;
    const bf16* base = qkv + (size_t)e * L * ld_qkv + col;
    bf16* dbase = dqkv + (size_t)e * L * ld_qkv + col;
    const bf16* dobase = d_out + (size_t)e * L * ld_out + col;

    float p[L][L];
    {
        uint4 q[L], k[L];
#pragma unroll
        for (int i = 0; i < L; i++) {
            q[i] = ld_nc16(base + (size_t)i * ld_qkv);
            k[i] = ld_nc16(base + (size_t)i * ld_qkv + H);
        }
#pragma unroll
        for (int i = 0; i < L; i++)
#pragma unroll
            for (int j = 0; j <= i; j++) p[i][j] = warp_sum(dot8(q[i], k[j])) * scale;
    }
    softmax_rows<L>(p);

    float ds[L][L];
    {
        uint4 dO[L], v[L];
#pragma unroll
        for (int i = 0; i < L; i++) {
            dO[i] = ld_nc16(dobase + (size_t)i * ld_out);
            v[i] = ld_nc16(base + (size_t)i * ld_qkv + 2 * H);
        }
        // dV[j] = sum_{i>=j} bf16(p_ij) dO[i]
#pragma unroll
        for (int j = 0; j < L; j++) {
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int i = j; i < L; i++) axpy8(acc, bf16_round(p[i][j]), dO[i]);
            *reinterpret_cast<uint4*>(dbase + (size_t)j * ld_qkv + 2 * H) = pack8(acc);
        }
#pragma unroll
        for (int i = 0; i < L; i++)
#pragma unroll
            for (int j = 0; j <= i; j++) ds[i][j] = warp_sum(dot8(dO[i], v[j]));   // dP_ij
    }
#pragma unroll
    for (int i = 0; i < L; i++) {
        float delta = 0.f;
#pragma unroll
        for (int j = 0; j <= i; j++) delta = fmaf(p[i][j], ds[i][j], delta);
#pragma unroll
        for (int j = 0; j <= i; j++) ds[i][j] = bf16_round(p[i][j] * (ds[i][j] - delta)) * scale;
    }
    {
        uint4 k[L];
#pragma unroll
        for (int i = 0; i < L; i++) k[i] = ld_nc16(base + (size_t)i * ld_qkv + H);
#pragma unroll
        for (int i = 0; i < L; i++) {   // dQ[i] = scale * sum_{j<=i} dS_ij k[j]
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int j = 0; j <= i; j++) axpy8(acc, ds[i][j], k[j]);
            if (rope_cos) rope_bwd_slice(acc, rope_cos, rope_sin, i, lane);
            *reinterpret_cast<uint4*>(dbase + (size_t)i * ld_qkv) = pack8(acc);
        }
    }
    {
        uint4 q[L];
#pragma unroll
        for (int i = 0; i < L; i++) q[i] = ld_nc16(base + (size_t)i * ld_qkv);
#pragma unroll
        for (int j = 0; j < L; j++) {   // dK[j] = scale * sum_{i>=j} dS_ij q[i]
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int i = j; i < L; i++) axpy8(acc, ds[i][j], q[i]);
            if (rope_cos) rope_bwd_slice(acc, rope_cos, rope_sin, j, lane);
            *reinterpret_cast<uint4*>(dbase + (size_t)j * ld_qkv + H) = pack8(acc);
        }
    }
}

}   // namespace

#define B200_TINY_DISPATCH(KERN, ...)                                                  \
    switch (L) {                                                                       \
        case 1: KERN<1><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 2: KERN<2><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 3: KERN<3><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 4: KERN<4><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 5: KERN<5><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 6: KERN<6><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        case 7: KERN<7><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break;  \
        default: KERN<8><<<grid, WARPS_PER_CTA * 32, 0, stream>>>(__VA_ARGS__); break; \
    }

// qkv: [n_events * L, ld_qkv] packed (q | k | v thirds of n_heads*256 columns, post-RoPE); out: [n_events * L, ld_out]
extern "C" int b200_attn_tiny_fwd(void* qkv, void* out, int n_events, int L, int n_heads, int head_dim, int ld_qkv,
                                  int ld_out, float scale, const void* rope_cos, const void* rope_sin, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == TD, "attn_tiny_fwd: head_dim %d unsupported (256 only)", head_dim);
    B200_CHECK_ARG(L >= 1 && L <= 8, "attn_tiny_fwd: L=%d outside 1..8", L);
    B200_CHECK_ARG(ld_qkv % 8 == 0 && ld_out % 8 == 0, "attn_tiny_fwd: leading dims must be multiples of 8");
    if (n_events == 0) return B200_OK;
    const int grid = (n_events * n_heads + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    B200_TINY_DISPATCH(tiny_attn_fwd_kernel, (bf16*)qkv, (bf16*)out, n_events, n_heads, ld_qkv, ld_out, scale,
                       (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_tiny_fwd");
    return B200_OK;
}

extern "C" int b200_attn_tiny_bwd(const void* qkv, const void* d_out, void* dqkv, int n_events, int L, int n_heads,
                                  int head_dim, int ld_qkv, int ld_out, float scale, const void* rope_cos,
                                  const void* rope_sin, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == TD, "attn_tiny_bwd: head_dim %d unsupported (256 only)", head_dim);
    B200_CHECK_ARG(L >= 1 && L <= 8, "attn_tiny_bwd: L=%d outside 1..8", L);
    B200_CHECK_ARG(ld_qkv % 8 == 0 && ld_out % 8 == 0, "attn_tiny_bwd: leading dims must be multiples of 8");
    if (n_events == 0) return B200_OK;
    const int grid = (n_events * n_heads + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    B200_TINY_DISPATCH(tiny_attn_bwd_kernel, (const bf16*)qkv, (const bf16*)d_out, (bf16*)dqkv, n_events, n_heads, ld_qkv,
                       ld_out, scale, (const bf16*)rope_cos, (const bf16*)rope_sin);
    B200_CHECK_LAUNCH("attn_tiny_bwd");
    return B200_OK;
}
