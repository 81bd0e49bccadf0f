// Rotary position embedding: the one definition of its arithmetic, its rounding points and the in-segment positions of
// ragged batches.  Every kernel that rotates q or k (the stand-alone RoPE kernel, the QKV GEMM epilogue, the token- and
// event-level attention, the decode kernels) computes through these functions, so fused and unfused paths agree bit for
// bit.  Each kernel keeps its own table loads and data layout; only the arithmetic lives here.
//
// hf modeling_llama.py:262-268 rotates the q and k projections with apply_rotary_pos_emb (:146-168):
// x * cos + rotate_half(x) * sin, rotate_half(x) = cat(-x2, x1) (:138-142).  On the (x1, x2) = (x[d], x[d + D/2]) pairs, with every
// op rounding to bf16 as the reference's eager bf16 path does:
//   forward : o1 = bf16(bf16(x1 c) + bf16(-x2 s)),  o2 = bf16(bf16(x2 c) + bf16(x1 s))   (three roundings)
//   backward: dx1 = d1 c + d2 s,  dx2 = d2 c - d1 s   (gradient w.r.t. the pre-rotation x: one rounding, on the store)
// The functions return the fp32 value before the last rounding: the caller rounds it on its bf16 store, or with
// bf16_round where the value stays in fp32.  Each expression is written once, so FMA contraction is the same everywhere.
#pragma once
#include "common.cuh"

// Forward rotation of one element x, given its partner (the other element of its pair), the pair's c, s and whether x
// is in the second half of the head.
__device__ __forceinline__ float rope_fwd_elem(float x, float partner, float c, float s, bool second_half) {
    return bf16_round(x * c) + bf16_round((second_half ? partner : -partner) * s);
}

// Backward rotation of one element x of the gradient, in the same form.
__device__ __forceinline__ float rope_bwd_elem(float x, float partner, float c, float s, bool second_half) {
    return second_half ? x * c - partner * s : x * c + partner * s;
}

// head_dim 256 across a warp, 8 elements per lane: lane l holds d = 8l .. 8l + 7, so its partners are in lane l ^ 16 and
// lanes 16..31 hold the second half.  c, s: the lane's 8 table entries (columns 8 (l % 16) .. of the [pos][128] tables).
// In place; the whole warp must call.
__device__ __forceinline__ void rope_fwd_lane(float* x, const float* c, const float* s, int lane) {
    const bool second_half = lane >= 16;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const float partner = __shfl_xor_sync(0xffffffffu, x[j], 16);
        x[j] = rope_fwd_elem(x[j], partner, c[j], s[j], second_half);
    }
}

__device__ __forceinline__ void rope_bwd_lane(float* x, const float* c, const float* s, int lane) {
    const bool second_half = lane >= 16;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const float partner = __shfl_xor_sync(0xffffffffu, x[j], 16);
        x[j] = rope_bwd_elem(x[j], partner, c[j], s[j], second_half);
    }
}

// Ragged batches: every sequence owns a segment of whole SEG_TILE-row tiles of the packed rows (the event-level
// attention's tile height, so no tile mixes sequences).  seg[2 t] / seg[2 t + 1] = first / last tile of tile t's
// segment.  A row's RoPE position counts from its segment's first row.
constexpr int SEG_TILE_LOG2 = 6;
constexpr int SEG_TILE = 1 << SEG_TILE_LOG2;

// first row of the segment that holds tile t
__device__ __forceinline__ int seg_first_row(const int* seg, int t) { return SEG_TILE * seg[2 * t]; }

// RoPE position of packed row r >= 0 (in tile r / SEG_TILE)
__device__ __forceinline__ int seg_pos(const int* seg, int r) { return r - seg_first_row(seg, r >> SEG_TILE_LOG2); }
