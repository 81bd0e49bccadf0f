// HBM-bound kernels of the MIDIModel hot path: embedding gather-sum (midi_model.py:145-146),
// inner-input builder (midi_model.py:126-131), RMSNorm (hf modeling_llama.py:62-67), RoPE
// (hf :124-168), SwiGLU (hf :183), and their backward passes.  All arithmetic is fp32 on
// bf16 storage with the reference's rounding points (DESIGN.md 3.3).  16-byte vector
// accesses, one 128-thread CTA per row (rows are 2 KB at hidden=1024), grids sized in rows.
#include "common.cuh"
#include "rope.cuh"
#include "../../include/midi_b200.h"

namespace {

constexpr int ROW_THREADS = 128;
constexpr int MAXV = 8;   // vectors of 8 bf16 per thread: hidden <= 128*8*8 = 8192

// ---------------------------------------------------------------------------
// embedding
// ---------------------------------------------------------------------------
// out[m, :] = bf16( sum_t fp32(table[ids[m, t], :]) )   -- one rounding (DESIGN.md 3.3)
__global__ void embed_sum_fwd_kernel(const long long* __restrict__ ids, const bf16* __restrict__ table,
                                     bf16* __restrict__ out, int T, int H, int V) {
    const int m = blockIdx.x;
    const long long* row_ids = ids + (size_t)m * T;
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int t = 0; t < T; t++) {
            long long id = row_ids[t];
            if (id < 0 || id >= V) continue;
            float f[8];
            unpack8(*reinterpret_cast<const uint4*>(table + (size_t)id * H + v * 8), f);
#pragma unroll
            for (int j = 0; j < 8; j++) acc[j] += f[j];
        }
        *reinterpret_cast<uint4*>(out + (size_t)m * H + v * 8) = pack8(acc);
    }
}

// out[(e*Tin + 0), :] = hidden[e, :] ; out[(e*Tin + j), :] = table[ids[e, j-1], :]   (cat([hidden, embed(x)]))
__global__ void inner_input_fwd_kernel(const bf16* __restrict__ hidden, const long long* __restrict__ ids,
                                       const bf16* __restrict__ table, bf16* __restrict__ out, int Tin, int n_ids,
                                       int has_hidden, int H, int V) {
    const int r = blockIdx.x;
    const int e = r / Tin, j = r % Tin;
    const bf16* src;
    if (has_hidden && j == 0) {
        src = hidden + (size_t)e * H;
    } else {
        long long id = ids[(size_t)e * n_ids + (j - has_hidden)];
        if (id < 0 || id >= V) id = 0;
        src = table + (size_t)id * H;
    }
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
        *reinterpret_cast<uint4*>(out + (size_t)r * H + v * 8) = *reinterpret_cast<const uint4*>(src + v * 8);
}

// dhidden[e,:] (+)= dx[e*Tin, :]
__global__ void inner_input_bwd_hidden_kernel(const bf16* __restrict__ dx, bf16* __restrict__ dhidden, int Tin, int H) {
    const int e = blockIdx.x;
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
        *reinterpret_cast<uint4*>(dhidden + (size_t)e * H + v * 8) =
            *reinterpret_cast<const uint4*>(dx + (size_t)e * Tin * H + v * 8);
}

// train.py --sample-seq (train.py:172-178): event n is event row rows[n] of hidden [n_rows, H] / y [n_rows, T].
// Block (n, j): out[n*T + j] = j == 0 ? hidden[rows[n]] : table[y[rows[n], j-1]], and y_sel[n, j] = y[rows[n], j].
// A row outside [0, n_rows) reads nothing: its input rows are zero and its labels -1 (ignored by the loss and the
// embedding backward).
__global__ void inner_input_rows_fwd_kernel(const bf16* __restrict__ hidden, const long long* __restrict__ y,
                                            const int* __restrict__ rows, const bf16* __restrict__ table,
                                            bf16* __restrict__ out, long long* __restrict__ y_sel, int n_rows, int T,
                                            int H, int V) {
    const int n = blockIdx.x / T, j = blockIdx.x % T;
    const int r = rows[n];
    const bool live = r >= 0 && r < n_rows;
    const bf16* src = nullptr;
    if (live) {
        if (j == 0) {
            src = hidden + (size_t)r * H;
        } else {
            long long id = y[(size_t)r * T + j - 1];
            if (id < 0 || id >= V) id = 0;
            src = table + (size_t)id * H;
        }
    }
    if (threadIdx.x == 0) y_sel[(size_t)n * T + j] = live ? y[(size_t)r * T + j] : -1;
    bf16* dst = out + ((size_t)n * T + j) * H;
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
        *reinterpret_cast<uint4*>(dst + v * 8) = live ? *reinterpret_cast<const uint4*>(src + v * 8) : make_uint4(0, 0, 0, 0);
}

// dhidden[r,:] = dx[inv[r]*Tin, :] for a selected row (inv[r] in [0, n_events)), zero for every other row: the full
// gradient of the event-level output in one pass.  Indices are unique, so every row is written exactly once.
__global__ void inner_input_rows_bwd_hidden_kernel(const bf16* __restrict__ dx, const int* __restrict__ inv,
                                                   bf16* __restrict__ dhidden, int n_events, int Tin, int H) {
    const int r = blockIdx.x;
    const int e = inv[r];
    const bool live = e >= 0 && e < n_events;
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
        *reinterpret_cast<uint4*>(dhidden + (size_t)r * H + v * 8) =
            live ? *reinterpret_cast<const uint4*>(dx + (size_t)e * Tin * H + v * 8) : make_uint4(0, 0, 0, 0);
}

// ---- embedding backward: counting sort of the ids, then one segment-sum per (id, slice) ----
// id i (flat index) reads gradient row  (i / per_row) * row_stride + (i % per_row) * row_inner + row_off
__global__ void embed_hist_kernel(const long long* __restrict__ ids, int n, int V, int* __restrict__ counts) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        long long id = ids[i];
        if (id >= 0 && id < V) atomicAdd(&counts[id], 1);
    }
}
__global__ void embed_scan_kernel(const int* __restrict__ counts, int* __restrict__ offsets, int V) {
    // single block exclusive scan; V <= 1024 * items
    __shared__ int sh[1024];
    const int items = (V + 1023) / 1024;
    const int base = threadIdx.x * items;
    int local = 0;
    for (int k = 0; k < items; k++)
        if (base + k < V) local += counts[base + k];
    sh[threadIdx.x] = local;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        int v = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
        __syncthreads();
        sh[threadIdx.x] += v;
        __syncthreads();
    }
    int run = sh[threadIdx.x] - local;
    for (int k = 0; k < items; k++)
        if (base + k < V) {
            offsets[base + k] = run;
            run += counts[base + k];
        }
    if (threadIdx.x == 1023) offsets[V] = sh[1023];
}
__global__ void embed_fill_kernel(const long long* __restrict__ ids, int n, int V, const int* __restrict__ offsets,
                                  int* __restrict__ cursor, int* __restrict__ sorted) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        long long id = ids[i];
        if (id >= 0 && id < V) {
            int pos = atomicAdd(&cursor[id], 1);
            sorted[offsets[id] + pos] = i;
        }
    }
}
// grid (V, SLICES): segment v (all occurrences of token id v) is cut into ceil(len / SEG_ROWS) <= SLICES slices; block
// (v, y) sums the entries y, y+n, ... of its slice set.  Short segments (the common case) have one slice and store their
// sum directly; only long ones (event-type ids, common values) combine partials with vector reds.  The previous version
// always used 32 slices and 8 scalar atomics per thread: 109k blocks x 1024 atomics dominated the kernel.
constexpr int SEG_ROWS = 48;
__global__ void embed_segsum_kernel(const int* __restrict__ offsets, const int* __restrict__ sorted,
                                    const bf16* __restrict__ dout, float* __restrict__ acc32, int H, int per_row,
                                    int row_stride, int row_inner, int row_off, int pad_id) {
    const int v = blockIdx.x;
    if (v == pad_id) return;   // padding_idx row receives zero gradient (hf nn.Embedding(padding_idx))
    const int beg = offsets[v], end = offsets[v + 1];
    const int len = end - beg;
    int n_slices = (len + SEG_ROWS - 1) / SEG_ROWS;
    if (n_slices > (int)gridDim.y) n_slices = gridDim.y;
    if ((int)blockIdx.y >= n_slices) return;       // also covers len == 0
    auto row_of = [&](int i) -> const bf16* {
        return dout + ((size_t)(i / per_row) * row_stride + (size_t)(i % per_row) * row_inner + row_off) * H;
    };
    for (int c = threadIdx.x; c < H / 8; c += blockDim.x) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        int j = beg + blockIdx.y;
        // four rows in flight per thread
        for (; j + 3 * n_slices < end; j += 4 * n_slices) {
            const int i0 = sorted[j], i1 = sorted[j + n_slices], i2 = sorted[j + 2 * n_slices], i3 = sorted[j + 3 * n_slices];
            const uint4 u0 = ld_nc16(row_of(i0) + c * 8), u1 = ld_nc16(row_of(i1) + c * 8);
            const uint4 u2 = ld_nc16(row_of(i2) + c * 8), u3 = ld_nc16(row_of(i3) + c * 8);
            float f0[8], f1[8], f2[8], f3[8];
            unpack8(u0, f0); unpack8(u1, f1); unpack8(u2, f2); unpack8(u3, f3);
#pragma unroll
            for (int k = 0; k < 8; k++) acc[k] += (f0[k] + f1[k]) + (f2[k] + f3[k]);
        }
        for (; j < end; j += n_slices) {
            float f[8];
            unpack8(ld_nc16(row_of(sorted[j]) + c * 8), f);
#pragma unroll
            for (int k = 0; k < 8; k++) acc[k] += f[k];
        }
        float* dst = acc32 + (size_t)v * H + c * 8;
        if (n_slices == 1) {
            *reinterpret_cast<float4*>(dst) = make_float4(acc[0], acc[1], acc[2], acc[3]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
        } else {
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(acc[0]), "f"(acc[1]), "f"(acc[2]), "f"(acc[3]) : "memory");
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4), "f"(acc[4]), "f"(acc[5]), "f"(acc[6]), "f"(acc[7]) : "memory");
        }
    }
}
__global__ void f32_to_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, size_t n, int accumulate) {
    size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const size_t stride = (size_t)gridDim.x * blockDim.x * 4;
    for (; i < n; i += stride) {
        float4 a = *reinterpret_cast<const float4*>(src + i);
        bf162* o = reinterpret_cast<bf162*>(dst + i);
        if (accumulate) {
            float2 o0 = __bfloat1622float2(o[0]), o1 = __bfloat1622float2(o[1]);
            a.x = bf16_round(a.x) + o0.x; a.y = bf16_round(a.y) + o0.y;
            a.z = bf16_round(a.z) + o1.x; a.w = bf16_round(a.w) + o1.y;
        }
        o[0] = __floats2bfloat162_rn(a.x, a.y);
        o[1] = __floats2bfloat162_rn(a.z, a.w);
    }
}

// ---------------------------------------------------------------------------
// RMSNorm
// ---------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float t = 0.f;
    const int nw = blockDim.x >> 5;
    for (int i = 0; i < nw; i++) t += sh[i];
    return t;
}

// y = w * bf16(x * rsqrt(mean(x^2) + eps))  -- two roundings (DESIGN.md 3.3)
template <int VPT>
__global__ void __launch_bounds__(ROW_THREADS)
rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                   float* __restrict__ rstd_out, int M, int H, float eps) {
    __shared__ float sh[8];
    const int nv = H / 8;
    for (int m = blockIdx.x; m < M; m += gridDim.x) {
        float xv[VPT][8];
        float ss = 0.f;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int v = threadIdx.x + k * ROW_THREADS;
            if (v < nv) {
                unpack8(ld_nc16(x + (size_t)m * H + v * 8), xv[k]);
#pragma unroll
                for (int j = 0; j < 8; j++) ss += xv[k][j] * xv[k][j];
            }
        }
        ss = block_sum(ss, sh);
        const float rstd = rsqrtf(ss / (float)H + eps);
        if (threadIdx.x == 0 && rstd_out) rstd_out[m] = rstd;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int v = threadIdx.x + k * ROW_THREADS;
            if (v < nv) {
                float wv[8], o[8];
                unpack8(*reinterpret_cast<const uint4*>(w + v * 8), wv);
#pragma unroll
                for (int j = 0; j < 8; j++) o[j] = wv[j] * bf16_round(xv[k][j] * rstd);
                *reinterpret_cast<uint4*>(y + (size_t)m * H + v * 8) = pack8(o);
            }
        }
    }
}

// dx = dres + rstd * (dn - n * mean(dn . n)),  dn = dy*w, n = x*rstd ;  dw_partial[block,:] = sum_rows dy * n
template <int VPT>
__global__ void __launch_bounds__(ROW_THREADS)
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
                   const float* __restrict__ rstd_in, const bf16* __restrict__ dres, bf16* __restrict__ dx,
                   float* __restrict__ dw_partial, int M, int H) {
    __shared__ float sh[8];
    const int nv = H / 8;
    float dwacc[VPT][8];
#pragma unroll
    for (int k = 0; k < VPT; k++)
#pragma unroll
        for (int j = 0; j < 8; j++) dwacc[k][j] = 0.f;
    for (int m = blockIdx.x; m < M; m += gridDim.x) {
        const float rstd = rstd_in[m];
        float nn[VPT][8], dn[VPT][8];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int v = threadIdx.x + k * ROW_THREADS;
            if (v < nv) {
                float xv[8], dyv[8], wv[8];
                unpack8(ld_nc16(x + (size_t)m * H + v * 8), xv);
                unpack8(ld_nc16(dy + (size_t)m * H + v * 8), dyv);
                unpack8(*reinterpret_cast<const uint4*>(w + v * 8), wv);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    nn[k][j] = xv[j] * rstd;
                    dn[k][j] = dyv[j] * wv[j];
                    dot += dn[k][j] * nn[k][j];
                    dwacc[k][j] += dyv[j] * nn[k][j];
                }
            }
        }
        dot = block_sum(dot, sh) / (float)H;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int v = threadIdx.x + k * ROW_THREADS;
            if (v < nv) {
                float o[8];
                if (dres) unpack8(ld_nc16(dres + (size_t)m * H + v * 8), o);
                else {
#pragma unroll
                    for (int j = 0; j < 8; j++) o[j] = 0.f;
                }
#pragma unroll
                for (int j = 0; j < 8; j++) o[j] += rstd * (dn[k][j] - nn[k][j] * dot);
                *reinterpret_cast<uint4*>(dx + (size_t)m * H + v * 8) = pack8(o);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < VPT; k++) {
        const int v = threadIdx.x + k * ROW_THREADS;
        if (v < nv) {
            float* dst = dw_partial + (size_t)blockIdx.x * H + v * 8;
#pragma unroll
            for (int j = 0; j < 8; j++) dst[j] = dwacc[k][j];
        }
    }
}
// ---- warp-per-row variants (hidden = 256 * VPT): no block barrier, reductions are 5 shuffles; each lane owns
// VPT 16-byte vectors of the row (coalesced 512 B per warp access).  These are the ones used at hidden = 1024.
constexpr int WR_WARPS = 8;        // forward
constexpr int WRB_WARPS = 4;       // backward (155 regs/thread at hidden=1024 -> 3 CTAs of 4 warps per SM)

// Registers are what bounds this kernel's memory parallelism (ncu, round 2: 80 registers -> 24 warps per SM, 75 % of the
// stall cycles on the long scoreboard, 0.53-0.68 of the copy bandwidth): the row is kept PACKED (bf16 pairs -- h is a bf16
// value, so nothing is lost), the norm weight is re-read from L1 instead of living in 32 fp32 registers, and the launch
// bound asks for four CTAs (32 warps) per SM.
template <int VPT>
__global__ void __launch_bounds__(WR_WARPS * 32, (VPT <= 4) ? 4 : 2)
rmsnorm_fwd_warp_kernel(const bf16* __restrict__ x, const bf16* __restrict__ res, const bf16* __restrict__ w,
                        bf16* __restrict__ h_out, bf16* __restrict__ y, float* __restrict__ rstd_out, int M, float eps) {
    B200_PDL_TRIGGER();
    constexpr int H = 256 * VPT;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    for (int m = blockIdx.x * WR_WARPS + warp; m < M; m += gridDim.x * WR_WARPS) {
        uint4 hp[VPT], rp[VPT];
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            hp[k] = ld_nc16(x + (size_t)m * H + (lane + k * 32) * 8);
            if (res) rp[k] = ld_nc16(res + (size_t)m * H + (lane + k * 32) * 8);
        }
        float ss = 0.f;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            float xv[8];
            unpack8(hp[k], xv);
            if (res) {   // fused residual add: h = bf16(x + res) is the new residual stream (hf :325 / :331)
                float rv[8];
                unpack8(rp[k], rv);
#pragma unroll
                for (int j = 0; j < 8; j++) xv[j] = bf16_round(xv[j] + rv[j]);
                hp[k] = pack8(xv);
                *reinterpret_cast<uint4*>(h_out + (size_t)m * H + (lane + k * 32) * 8) = hp[k];
            }
#pragma unroll
            for (int j = 0; j < 8; j++) ss = fmaf(xv[j], xv[j], ss);
        }
        ss = warp_sum(ss);
        const float rstd = rsqrtf(ss / (float)H + eps);
        if (lane == 0 && rstd_out) rstd_out[m] = rstd;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            float xv[8], wv[8], o[8];
            unpack8(hp[k], xv);
            unpack8(*reinterpret_cast<const uint4*>(w + (lane + k * 32) * 8), wv);
#pragma unroll
            for (int j = 0; j < 8; j++) o[j] = wv[j] * bf16_round(xv[j] * rstd);
            *reinterpret_cast<uint4*>(y + (size_t)m * H + (lane + k * 32) * 8) = pack8(o);
        }
    }
}

// (Same register diet as the forward kernel: x and dy stay packed between the two passes and n = x*rstd, dn = dy*w are
// recomputed -- identical fp32 operations -- instead of living in 64 fp32 registers; the norm weight is re-read from L1.
// 157 -> ~100 registers, 3 -> 5 CTAs of 4 warps per SM.)
template <int VPT>
__global__ void __launch_bounds__(WRB_WARPS * 32, (VPT <= 4) ? 4 : 2)
rmsnorm_bwd_warp_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
                        const float* __restrict__ rstd_in, const bf16* __restrict__ dres, bf16* __restrict__ dx,
                        float* __restrict__ dw_acc, unsigned int* __restrict__ dw_ticket, bf16* __restrict__ dw,
                        int accumulate_dw, int M) {
    B200_PDL_TRIGGER();
    constexpr int H = 256 * VPT;
    extern __shared__ float wr_smem[];   // [WRB_WARPS][H]
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    float dwacc[VPT][8];
#pragma unroll
    for (int k = 0; k < VPT; k++)
#pragma unroll
        for (int j = 0; j < 8; j++) dwacc[k][j] = 0.f;
    for (int m = blockIdx.x * WRB_WARPS + warp; m < M; m += gridDim.x * WRB_WARPS) {
        uint4 xp[VPT], dyp[VPT], rp[VPT];
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            xp[k] = ld_nc16(x + (size_t)m * H + (lane + k * 32) * 8);
            dyp[k] = ld_nc16(dy + (size_t)m * H + (lane + k * 32) * 8);
            if (dres) rp[k] = ld_nc16(dres + (size_t)m * H + (lane + k * 32) * 8);
        }
        const float rstd = rstd_in[m];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            float xv[8], dyv[8], wv[8];
            unpack8(xp[k], xv);
            unpack8(dyp[k], dyv);
            unpack8(*reinterpret_cast<const uint4*>(w + (lane + k * 32) * 8), wv);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float nn = xv[j] * rstd;
                const float dn = dyv[j] * wv[j];
                dot = fmaf(dn, nn, dot);
                dwacc[k][j] = fmaf(dyv[j], nn, dwacc[k][j]);
            }
        }
        dot = warp_sum(dot) / (float)H;
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            float o[8], xv[8], dyv[8], wv[8];
            if (dres) unpack8(rp[k], o);
            else {
#pragma unroll
                for (int j = 0; j < 8; j++) o[j] = 0.f;
            }
            unpack8(xp[k], xv);
            unpack8(dyp[k], dyv);
            unpack8(*reinterpret_cast<const uint4*>(w + (lane + k * 32) * 8), wv);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float nn = xv[j] * rstd;
                const float dn = dyv[j] * wv[j];
                o[j] += rstd * (dn - nn * dot);
            }
            *reinterpret_cast<uint4*>(dx + (size_t)m * H + (lane + k * 32) * 8) = pack8(o);
        }
    }
    // weight gradient: the warps' partials meet in shared memory, the CTA adds its column sums to ONE fp32 accumulator row
    // in global memory (red.add), and the last CTA to finish (atomic ticket) rounds the row into dw and hands the
    // accumulator back zeroed -- no second launch for the column sum (it was 32 launches, 0.35 ms per step).  The
    // accumulation order over CTAs is not fixed; dw is a [H] vector whose fp32 sum is rounded to bf16 once.
    if (dw == nullptr) return;
#pragma unroll
    for (int k = 0; k < VPT; k++)
#pragma unroll
        for (int j = 0; j < 8; j++) wr_smem[warp * H + (lane + k * 32) * 8 + j] = dwacc[k][j];
    __syncthreads();
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
        float t = 0.f;
#pragma unroll
        for (int wi = 0; wi < WRB_WARPS; wi++) t += wr_smem[wi * H + c];
        atomicAdd(dw_acc + c, t);
    }
    __threadfence();
    __syncthreads();
    __shared__ int s_last;
    if (threadIdx.x == 0) s_last = (atomicAdd(dw_ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (int c = threadIdx.x; c < H; c += blockDim.x) {
            float t = __ldcg(dw_acc + c);
            if (accumulate_dw) t = bf16_round(t) + __bfloat162float(dw[c]);
            dw[c] = __float2bfloat16_rn(t);
            dw_acc[c] = 0.f;
        }
        if (threadIdx.x == 0) *dw_ticket = 0u;
    }
}

__global__ void colsum_partial_kernel(const float* __restrict__ partial, int nparts, int H, bf16* __restrict__ out,
                                      int accumulate) {
    // block (32, 8): x = column inside a 32-column tile, y = slice of the partial rows
    __shared__ float sh[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float s = 0.f;
    if (c < H)
        for (int p = threadIdx.y; p < nparts; p += 8) s += partial[(size_t)p * H + c];
    sh[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < H) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) t += sh[i][threadIdx.x];
        if (accumulate) t = bf16_round(t) + __bfloat162float(out[c]);
        out[c] = __float2bfloat16_rn(t);
    }
}

// ---------------------------------------------------------------------------
// RoPE
// ---------------------------------------------------------------------------
// cos/sin tables exactly as hf :124-135: fp32 pos * fp32(inv_freq buffer), fp32 cos/sin, cast to bf16.
__global__ void rope_table_kernel(const float* __restrict__ inv_freq, int half, int n_pos, int pos0, const int* pos0_dev,
                                  bf16* __restrict__ cos_t, bf16* __restrict__ sin_t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pos * half) return;
    const int s = i / half, j = i % half;
    const int base = pos0_dev ? *pos0_dev : pos0;
    const float f = (float)(base + s) * inv_freq[j];
    cos_t[i] = __float2bfloat16_rn(cosf(f));
    sin_t[i] = __float2bfloat16_rn(sinf(f));
}

// In place on the q and k thirds of packed qkv rows [rows, 3*H]; position of row r = pos0 (+ *pos0_dev) + r % S
// (the tables cover absolute positions), or its in-segment position with a segment table (rope.cuh).  RAGGED: row r of
// sequence r / S is at pos0 (+ *pos0_dev) + row_off[r / S] + r % S.
template <bool BWD, bool RAGGED = false>
__global__ void rope_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                            int rows, int S, int H, int D, int ld, int pos0, const int* __restrict__ pos0_dev,
                            const int* __restrict__ seg, const int* __restrict__ row_off) {
    const int r = blockIdx.x;
    int s;
    if constexpr (RAGGED) s = pos0 + (pos0_dev ? *pos0_dev : 0) + row_off[r / S] + r % S;
    else s = seg ? seg_pos(seg, r) : pos0 + (pos0_dev ? *pos0_dev : 0) + r % S;
    const int half = D / 2;
    const int vec_per_head = half / 8;
    const int heads2 = 2 * (H / D);   // q heads then k heads (k third starts at column H)
    const int total = heads2 * vec_per_head;
    bf16* row = qkv + (size_t)r * ld;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int hh = i / vec_per_head, v = i % vec_per_head;
        bf16* p1 = row + (size_t)hh * D + v * 8;   // q heads occupy [0,H), k heads [H,2H): contiguous in hh*D
        bf16* p2 = p1 + half;
        float x1[8], x2[8], c[8], sn[8], o1[8], o2[8];
        unpack8(*reinterpret_cast<const uint4*>(p1), x1);
        unpack8(*reinterpret_cast<const uint4*>(p2), x2);
        unpack8(*reinterpret_cast<const uint4*>(cos_t + (size_t)s * half + v * 8), c);
        unpack8(*reinterpret_cast<const uint4*>(sin_t + (size_t)s * half + v * 8), sn);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (!BWD) {
                o1[j] = rope_fwd_elem(x1[j], x2[j], c[j], sn[j], false);
                o2[j] = rope_fwd_elem(x2[j], x1[j], c[j], sn[j], true);
            } else {
                o1[j] = rope_bwd_elem(x1[j], x2[j], c[j], sn[j], false);
                o2[j] = rope_bwd_elem(x2[j], x1[j], c[j], sn[j], true);
            }
        }
        *reinterpret_cast<uint4*>(p1) = pack8(o1);
        *reinterpret_cast<uint4*>(p2) = pack8(o2);
    }
}

// ---------------------------------------------------------------------------
// SwiGLU on packed [rows, 2*I] = [gate | up]
// ---------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return sigmoid_f(x); }

// act = bf16( bf16(silu(g)) * u )   (two roundings, A.6)
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ act, size_t rows, int I) {
    const size_t nvec = rows * (size_t)(I / 8);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / (I / 8);
        const int c = (int)(i % (I / 8)) * 8;
        float g[8], u[8], o[8];
        unpack8(ld_nc16(gu + r * 2 * I + c), g);
        unpack8(ld_nc16(gu + r * 2 * I + I + c), u);
#pragma unroll
        for (int j = 0; j < 8; j++) o[j] = bf16_round(silu_f(g[j])) * u[j];
        *reinterpret_cast<uint4*>(act + r * I + c) = pack8(o);
    }
}
// y = bf16(x * s): the LoRA scaling lora_alpha / r applied to the rank-r down-projection and to its gradient
// (peft lora/layer.py Linear.forward: `lora_B(lora_A(x)) * scaling`); 16-byte vectors, scalar tail
__global__ void scale_bf16_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, size_t n, float s) {
    const size_t nvec = n / 8;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        float v[8];
        unpack8(ld_nc16(x + i * 8), v);
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] *= s;
        *reinterpret_cast<uint4*>(y + i * 8) = pack8(v);
    }
    if (blockIdx.x == 0)
        for (size_t i = nvec * 8 + threadIdx.x; i < n; i += blockDim.x)
            y[i] = __float2bfloat16_rn(__bfloat162float(x[i]) * s);
}
// dg = dact * u * silu'(g), du = dact * silu(g)
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ gu, const bf16* __restrict__ dact, bf16* __restrict__ dgu,
                                  size_t rows, int I) {
    B200_PDL_TRIGGER();
    const size_t nvec = rows * (size_t)(I / 8);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / (I / 8);
        const int c = (int)(i % (I / 8)) * 8;
        float g[8], u[8], d[8], dg[8], du[8];
        unpack8(ld_nc16(gu + r * 2 * I + c), g);
        unpack8(ld_nc16(gu + r * 2 * I + I + c), u);
        unpack8(ld_nc16(dact + r * I + c), d);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float sg = sigmoidf_(g[j]);
            const float silu = g[j] * sg;
            dg[j] = d[j] * u[j] * (sg * (1.f + g[j] * (1.f - sg)));
            du[j] = d[j] * silu;
        }
        *reinterpret_cast<uint4*>(dgu + r * 2 * I + c) = pack8(dg);
        *reinterpret_cast<uint4*>(dgu + r * 2 * I + I + c) = pack8(du);
    }
}

inline int grid_for(size_t n_items, int threads, int per_sm = 16) {
    size_t b = (n_items + threads - 1) / threads;
    size_t cap = (size_t)b200_num_sms() * per_sm;
    return (int)(b < cap ? (b ? b : 1) : cap);
}

}   // namespace

// ===========================================================================
// C ABI
// ===========================================================================
extern "C" int b200_embed_sum_fwd(const long long* ids, const void* table, void* out, int M, int T, int H, int V,
                                  cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0 && M >= 0, "embed_sum_fwd: H must be a multiple of 8");
    if (M == 0) return B200_OK;
    embed_sum_fwd_kernel<<<M, ROW_THREADS, 0, stream>>>(ids, (const bf16*)table, (bf16*)out, T, H, V);
    B200_CHECK_LAUNCH("embed_sum_fwd");
    return B200_OK;
}

extern "C" int b200_inner_input_fwd(const void* hidden, const long long* ids, const void* table, void* out, int n_events,
                                    int n_ids, int H, int V, cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0, "inner_input_fwd: H must be a multiple of 8");
    const int has_hidden = hidden != nullptr;
    const int Tin = n_ids + has_hidden;
    if (n_events == 0 || Tin == 0) return B200_OK;
    inner_input_fwd_kernel<<<n_events * Tin, ROW_THREADS, 0, stream>>>((const bf16*)hidden, ids, (const bf16*)table,
                                                                       (bf16*)out, Tin, n_ids, has_hidden, H, V);
    B200_CHECK_LAUNCH("inner_input_fwd");
    return B200_OK;
}

extern "C" int b200_inner_input_bwd_hidden(const void* dx, void* dhidden, int n_events, int Tin, int H,
                                           cudaStream_t stream) {
    if (n_events == 0) return B200_OK;
    inner_input_bwd_hidden_kernel<<<n_events, ROW_THREADS, 0, stream>>>((const bf16*)dx, (bf16*)dhidden, Tin, H);
    B200_CHECK_LAUNCH("inner_input_bwd_hidden");
    return B200_OK;
}

extern "C" int b200_inner_input_rows_fwd(const void* hidden, const long long* y, const int* rows, const void* table,
                                         void* out, long long* y_sel, int n_events, int n_rows, int T, int H, int V,
                                         cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0, "inner_input_rows_fwd: H must be a multiple of 8");
    B200_CHECK_ARG(n_events >= 0 && n_rows >= 0 && T >= 1 && V >= 1,
                   "inner_input_rows_fwd: bad sizes (n_events %d, n_rows %d, T %d, V %d)", n_events, n_rows, T, V);
    B200_CHECK_ARG(n_events == 0 || (hidden && y && rows && table && out && y_sel),
                   "inner_input_rows_fwd: null pointer");
    B200_CHECK_ARG((long long)n_events * T <= 0x7fffffffLL, "inner_input_rows_fwd: too many rows");
    if (n_events == 0) return B200_OK;
    inner_input_rows_fwd_kernel<<<n_events * T, ROW_THREADS, 0, stream>>>((const bf16*)hidden, y, rows,
                                                                          (const bf16*)table, (bf16*)out, y_sel, n_rows,
                                                                          T, H, V);
    B200_CHECK_LAUNCH("inner_input_rows_fwd");
    return B200_OK;
}

extern "C" int b200_inner_input_rows_bwd_hidden(const void* dx, const int* inv, void* dhidden, int n_rows, int n_events,
                                                int Tin, int H, cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0, "inner_input_rows_bwd_hidden: H must be a multiple of 8");
    B200_CHECK_ARG(n_rows >= 0 && n_events >= 0 && Tin >= 1,
                   "inner_input_rows_bwd_hidden: bad sizes (n_rows %d, n_events %d, Tin %d)", n_rows, n_events, Tin);
    B200_CHECK_ARG(n_rows == 0 || (inv && dhidden && (dx || n_events == 0)), "inner_input_rows_bwd_hidden: null pointer");
    if (n_rows == 0) return B200_OK;
    inner_input_rows_bwd_hidden_kernel<<<n_rows, ROW_THREADS, 0, stream>>>((const bf16*)dx, inv, (bf16*)dhidden,
                                                                           n_events, Tin, H);
    B200_CHECK_LAUNCH("inner_input_rows_bwd_hidden");
    return B200_OK;
}

// Host data path (train.py:71,168-176): the dataset keeps token matrices as int16; one launch widens a [B, S+1, T] int16
// batch and cuts it into the two contiguous int64 views the step needs, x = batch[:, :-1] and y = batch[:, 1:].
namespace {
__global__ void batch_to_xy_kernel(const short* __restrict__ b, long long* __restrict__ x, long long* __restrict__ y,
                                   long long n, int S, int T) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long per = (long long)S * T;
        const long long bi = i / per, rem = i - bi * per;
        const short* src = b + bi * (per + T) + rem;
        x[i] = src[0];
        y[i] = src[T];
    }
}
}   // namespace

extern "C" int b200_batch_to_xy_i16(const void* batch, int B, int S1, int T, long long* x, long long* y, cudaStream_t stream) {
    B200_CHECK_ARG(B >= 0 && S1 >= 1 && T >= 1, "batch_to_xy: bad shape (%d, %d, %d)", B, S1, T);
    const long long n = (long long)B * (S1 - 1) * T;
    if (n == 0) return B200_OK;
    batch_to_xy_kernel<<<grid_for((size_t)n, 256), 256, 0, stream>>>((const short*)batch, x, y, n, S1 - 1, T);
    B200_CHECK_LAUNCH("batch_to_xy");
    return B200_OK;
}

// The same widening into a ragged (segment-packed) layout: packed row r takes x from batch row src[r] and y from the row
// after it (src[r] indexes the B * S1 rows of the batch), or pad_id in every column when src[r] < 0 (a gap row).  Only
// rows named by src and the row after each are read.
namespace {
__global__ void batch_to_xy_packed_kernel(const short* __restrict__ b, const int* __restrict__ src, long long* __restrict__ x,
                                          long long* __restrict__ y, long long n, int T, int pad_id) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / T;
        const int c = (int)(i - r * T);
        const int s = src[r];
        if (s < 0) {
            x[i] = pad_id;
            y[i] = pad_id;
        } else {
            const short* p = b + (long long)s * T + c;
            x[i] = p[0];
            y[i] = p[T];
        }
    }
}
}   // namespace

extern "C" int b200_batch_to_xy_packed_i16(const void* batch, int T, const int* src, int n_rows, int pad_id, long long* x,
                                           long long* y, cudaStream_t stream) {
    B200_CHECK_ARG(T >= 1 && n_rows >= 0 && (n_rows == 0 || src), "batch_to_xy_packed: bad arguments (T %d, rows %d)", T,
                   n_rows);
    const long long n = (long long)n_rows * T;
    if (n == 0) return B200_OK;
    batch_to_xy_packed_kernel<<<grid_for((size_t)n, 256), 256, 0, stream>>>((const short*)batch, src, x, y, n, T, pad_id);
    B200_CHECK_LAUNCH("batch_to_xy_packed");
    return B200_OK;
}

// train.py's augmentation (MIDITokenizerV2.augment, midi_tokenizer.py:1023-1102) of a cropped int16 batch, in place, one
// thread per token row.  The host draws the shifts and decides the two rules that need the whole file (corpus metadata):
// whether any non-drum note would leave 0..127 (then the sample is skipped entirely) and which tracks are drum-only.
// Python's % is floored and the pitch / sf operands can be negative, hence floor_mod.  Zero shifts still clamp.
namespace {
__device__ __forceinline__ int floor_mod(int a, int m) {
    const int r = a % m;
    return r < 0 ? r + m : r;
}

__device__ __forceinline__ int clamp_i(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void augment_kernel(short* __restrict__ b, const int* __restrict__ aug, long long n_rows, int L, int T,
                               b200_augment_ids id) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (long long)gridDim.x * blockDim.x) {
        const int* a = aug + (r / L) * B200_AUG_COLS;
        if (a[B200_AUG_SKIP]) continue;
        short* t = b + r * T;
        const int ev = t[0];
        if (ev == id.note || ev == id.patch_change || ev == id.control_change) {
            // every v2 event with a channel has it at position 4
            const int s = a[B200_AUG_CHANNEL];
            const int c0 = t[4] - id.channel;
            int c = floor_mod(c0 + s, 16);
            if (c0 == 9) c = 9;
            else if (c == 9) c = floor_mod(9 + s, 16);
            t[4] = (short)(id.channel + c);
            if (ev == id.note) {
                int p = t[5] - id.pitch;
                if (c0 != 9) p += a[B200_AUG_PITCH];
                t[5] = (short)(id.pitch + p);
                t[6] = (short)(id.velocity + clamp_i(t[6] - id.velocity + a[B200_AUG_VELOCITY], 1, 127));
            } else if (ev == id.control_change) {
                const int cc = t[5] - id.controller;
                if (cc == 1 || cc == 2 || cc == 7 || cc == 11)
                    t[6] = (short)(id.value + clamp_i(t[6] - id.value + a[B200_AUG_CC_VALUE], 1, 127));
            }
        } else if (ev == id.set_tempo) {
            t[4] = (short)(id.bpm + clamp_i(t[4] - id.bpm + a[B200_AUG_BPM], 1, 383));
        } else if (ev == id.key_signature) {
            const int tr = t[3] - id.track;
            const int mi = t[5] - id.mi;
            const int k = floor_mod(floor_mod((t[4] - id.sf - 7) * 7, 12) + a[B200_AUG_PITCH], 12);   // sf2key, shift
            int sf = (k * 7) % 12;                                                                    // key2sf
            if (sf > 6 || (mi == 1 && sf >= 5)) sf -= 12;
            if (tr >= 0 && tr < 128 && ((unsigned)a[B200_AUG_DRUM + (tr >> 5)] >> (tr & 31) & 1u)) sf = 0;
            t[4] = (short)(id.sf + sf + 7);
        }
    }
}
}   // namespace

extern "C" int b200_augment_i16(void* batch, int B, int L, int T, const int* aug, const b200_augment_ids* ids,
                                cudaStream_t stream) {
    B200_CHECK_ARG(B >= 0 && L >= 0 && T >= 7, "augment: bad shape (%d, %d, %d)", B, L, T);
    B200_CHECK_ARG(ids != nullptr, "augment: null id table");
    const long long n = (long long)B * L;
    if (n == 0) return B200_OK;
    B200_CHECK_ARG(batch && aug, "augment: null pointer");
    augment_kernel<<<grid_for((size_t)n, 256), 256, 0, stream>>>((short*)batch, aug, n, L, T, *ids);
    B200_CHECK_LAUNCH("augment");
    return B200_OK;
}

extern "C" size_t b200_embed_bwd_workspace_bytes(int n_ids, int V, int H) {
    return (size_t)(3 * (V + 1) + n_ids) * sizeof(int) + 256 + (size_t)V * H * sizeof(float);
}

// dtable[v,:] (+)= sum over ids i == v of dout[row(i), :]; padding row gets zero (or is left untouched when accumulating)
extern "C" int b200_embed_bwd(const long long* ids, int n_ids, const void* dout, void* dtable, int V, int H, int per_row,
                              int row_stride, int row_inner, int row_off, int pad_id, int accumulate, void* workspace,
                              size_t workspace_bytes, cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0, "embed_bwd: H must be a multiple of 8");
    B200_CHECK_ARG(workspace_bytes >= b200_embed_bwd_workspace_bytes(n_ids, V, H), "embed_bwd: workspace too small");
    B200_CHECK_ARG(V <= 1024 * 64, "embed_bwd: vocabulary too large");
    int* counts = (int*)workspace;
    int* offsets = counts + (V + 1);
    int* cursor = offsets + (V + 1);
    int* sorted = cursor + (V + 1);
    float* acc32 = (float*)(((uintptr_t)(sorted + n_ids) + 255) & ~(uintptr_t)255);
    B200_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 3 * (V + 1), stream), "embed_bwd memset");
    B200_CUDA(cudaMemsetAsync(acc32, 0, sizeof(float) * (size_t)V * H, stream), "embed_bwd memset");
    if (n_ids > 0) {
        const int g = grid_for(n_ids, 256);
        embed_hist_kernel<<<g, 256, 0, stream>>>(ids, n_ids, V, counts);
        embed_scan_kernel<<<1, 1024, 0, stream>>>(counts, offsets, V);
        embed_fill_kernel<<<g, 256, 0, stream>>>(ids, n_ids, V, offsets, cursor, sorted);
        dim3 grid(V, 32);
        embed_segsum_kernel<<<grid, ROW_THREADS, 0, stream>>>(offsets, sorted, (const bf16*)dout, acc32, H, per_row,
                                                              row_stride, row_inner, row_off, pad_id);
        B200_COUNT_EXTRA(4);
    }
    const size_t n = (size_t)V * H;
    f32_to_bf16_kernel<<<grid_for(n / 4, 256), 256, 0, stream>>>(acc32, (bf16*)dtable, n, accumulate);
    B200_CHECK_LAUNCH("embed_bwd");
    return B200_OK;
}

static int rmsnorm_fwd_impl(const void* x, const void* res, const void* w, void* h_out, void* y, float* rstd, int M, int H,
                            float eps, cudaStream_t stream);

extern "C" int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int H, float eps,
                                cudaStream_t stream) {
    return rmsnorm_fwd_impl(x, nullptr, w, nullptr, y, rstd, M, H, eps, stream);
}

// h = bf16(x + res) (the residual add of hf modeling_llama.py:325 / :331, written to h_out) ; y = RMSNorm(h) * w
extern "C" int b200_add_rmsnorm_fwd(const void* x, const void* res, const void* w, void* h_out, void* y, float* rstd, int M,
                                    int H, float eps, cudaStream_t stream) {
    B200_CHECK_ARG(H == 256 || H == 512 || H == 1024 || H == 2048, "add_rmsnorm_fwd: hidden size %d unsupported", H);
    B200_CHECK_ARG(res != nullptr && h_out != nullptr, "add_rmsnorm_fwd: res and h_out are required");
    return rmsnorm_fwd_impl(x, res, w, h_out, y, rstd, M, H, eps, stream);
}

static int rmsnorm_fwd_impl(const void* x, const void* res, const void* w, void* h_out, void* y, float* rstd, int M, int H,
                            float eps, cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0 && H <= ROW_THREADS * 8 * MAXV, "rmsnorm_fwd: unsupported hidden size %d", H);
    if (M == 0) return B200_OK;
    if (H == 256 || H == 512 || H == 1024 || H == 2048) {
        int g = (M + WR_WARPS - 1) / WR_WARPS;
        const int cap = b200_num_sms() * 8;
        if (g > cap) g = cap;
#define B200_RMS_FWDW(V) rmsnorm_fwd_warp_kernel<V><<<g, WR_WARPS * 32, 0, stream>>>((const bf16*)x, (const bf16*)res, (const bf16*)w, (bf16*)h_out, (bf16*)y, rstd, M, eps)
        if (H == 256) B200_RMS_FWDW(1); else if (H == 512) B200_RMS_FWDW(2); else if (H == 1024) B200_RMS_FWDW(4); else B200_RMS_FWDW(8);
#undef B200_RMS_FWDW
        B200_CHECK_LAUNCH("rmsnorm_fwd");
        return B200_OK;
    }
    const int grid = M < b200_num_sms() * 16 ? M : b200_num_sms() * 16;
    const int vpt = (H / 8 + ROW_THREADS - 1) / ROW_THREADS;
#define B200_RMS_FWD(V) rmsnorm_fwd_kernel<V><<<grid, ROW_THREADS, 0, stream>>>((const bf16*)x, (const bf16*)w, (bf16*)y, rstd, M, H, eps)
    if (vpt <= 1) B200_RMS_FWD(1); else if (vpt <= 2) B200_RMS_FWD(2); else if (vpt <= 4) B200_RMS_FWD(4); else B200_RMS_FWD(8);
#undef B200_RMS_FWD
    B200_CHECK_LAUNCH("rmsnorm_fwd");
    return B200_OK;
}

extern "C" int b200_rmsnorm_bwd_parts(void) { return b200_num_sms() * 4; }

// workspace: float[b200_rmsnorm_bwd_parts() * H]
extern "C" int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres,
                                void* dx, void* dw, int M, int H, int accumulate_dw, void* workspace,
                                size_t workspace_bytes, cudaStream_t stream) {
    B200_CHECK_ARG(H % 8 == 0 && H <= ROW_THREADS * 8 * MAXV, "rmsnorm_bwd: unsupported hidden size %d", H);
    const int parts = b200_rmsnorm_bwd_parts();
    B200_CHECK_ARG(workspace_bytes >= (size_t)parts * H * sizeof(float), "rmsnorm_bwd: workspace too small");
    if (M == 0) {   // no rows: the column sum is zero
        if (dw && !accumulate_dw) B200_CUDA(cudaMemsetAsync(dw, 0, (size_t)H * sizeof(bf16), stream), "rmsnorm_bwd dw");
        return B200_OK;
    }
    if (H == 256 || H == 512 || H == 1024) {
        int g = (M + WRB_WARPS - 1) / WRB_WARPS;
        if (g > parts) g = parts;
        const size_t smem = (size_t)WRB_WARPS * H * sizeof(float);
#define B200_RMS_BWDW(V)                                                                                              \
    do {                                                                                                              \
        static bool cfg = false;                                                                                      \
        if (!cfg) {                                                                                                   \
            B200_CUDA(cudaFuncSetAttribute(rmsnorm_bwd_warp_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                           (int)smem), "rmsnorm_bwd smem");                                           \
            cfg = true;                                                                                               \
        }                                                                                                             \
        rmsnorm_bwd_warp_kernel<V><<<g, WRB_WARPS * 32, smem, stream>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, \
                                                                       rstd, (const bf16*)dres, (bf16*)dx,            \
                                                                       (float*)workspace, (unsigned int*)((float*)workspace + H), \
                                                                       (bf16*)dw, accumulate_dw, M);                  \
    } while (0)
        if (H == 256) B200_RMS_BWDW(1); else if (H == 512) B200_RMS_BWDW(2); else B200_RMS_BWDW(4);
#undef B200_RMS_BWDW
        B200_CHECK_LAUNCH("rmsnorm_bwd");
        return B200_OK;
    }
    const int vpt = (H / 8 + ROW_THREADS - 1) / ROW_THREADS;
#define B200_RMS_BWD(V) rmsnorm_bwd_kernel<V><<<parts, ROW_THREADS, 0, stream>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, rstd, (const bf16*)dres, (bf16*)dx, (float*)workspace, M, H)
    if (vpt <= 1) B200_RMS_BWD(1); else if (vpt <= 2) B200_RMS_BWD(2); else if (vpt <= 4) B200_RMS_BWD(4); else B200_RMS_BWD(8);
#undef B200_RMS_BWD
    B200_CHECK_LAUNCH("rmsnorm_bwd");
    if (dw) {
        colsum_partial_kernel<<<(H + 31) / 32, dim3(32, 8), 0, stream>>>((const float*)workspace, parts, H, (bf16*)dw,
                                                                        accumulate_dw);
        B200_CHECK_LAUNCH("rmsnorm_bwd_dw");
    }
    // the partials overwrote the warp kernels' accumulator row and ticket: hand the workspace back zeroed, as they do
    B200_CUDA(cudaMemsetAsync(workspace, 0, (size_t)parts * H * sizeof(float), stream), "rmsnorm_bwd workspace");
    return B200_OK;
}

extern "C" int b200_rope_table(const float* inv_freq, int half, int n_pos, int pos0, const int* pos0_dev, void* cos_t,
                               void* sin_t, cudaStream_t stream) {
    if (n_pos <= 0) return B200_OK;
    const int n = n_pos * half;
    rope_table_kernel<<<(n + 255) / 256, 256, 0, stream>>>(inv_freq, half, n_pos, pos0, pos0_dev, (bf16*)cos_t,
                                                          (bf16*)sin_t);
    B200_CHECK_LAUNCH("rope_table");
    return B200_OK;
}

extern "C" int b200_rope_qk(void* qkv, const void* cos_t, const void* sin_t, int rows, int S, int H, int D, int ld,
                            int backward, int pos0, const int* pos0_dev, cudaStream_t stream) {
    B200_CHECK_ARG(D % 16 == 0 && H % D == 0 && ld % 8 == 0, "rope: head_dim must be a multiple of 16");
    if (rows == 0) return B200_OK;
    if (backward)
        rope_kernel<true><<<rows, ROW_THREADS, 0, stream>>>((bf16*)qkv, (const bf16*)cos_t, (const bf16*)sin_t, rows, S, H, D, ld, pos0, pos0_dev, nullptr, nullptr);
    else
        rope_kernel<false><<<rows, ROW_THREADS, 0, stream>>>((bf16*)qkv, (const bf16*)cos_t, (const bf16*)sin_t, rows, S, H, D, ld, pos0, pos0_dev, nullptr, nullptr);
    B200_CHECK_LAUNCH("rope");
    return B200_OK;
}

extern "C" int b200_rope_qk_seg(void* qkv, const void* cos_t, const void* sin_t, int rows, const int* seg, int H, int D,
                                int ld, int backward, cudaStream_t stream) {
    B200_CHECK_ARG(D % 16 == 0 && H % D == 0 && ld % 8 == 0, "rope_seg: head_dim must be a multiple of 16");
    B200_CHECK_ARG(rows % SEG_TILE == 0 && (rows == 0 || seg), "rope_seg: rows (%d) must be whole 64-row tiles of a segment table",
                   rows);
    if (rows == 0) return B200_OK;
    if (backward)
        rope_kernel<true><<<rows, ROW_THREADS, 0, stream>>>((bf16*)qkv, (const bf16*)cos_t, (const bf16*)sin_t, rows, 1, H, D, ld, 0, nullptr, seg, nullptr);
    else
        rope_kernel<false><<<rows, ROW_THREADS, 0, stream>>>((bf16*)qkv, (const bf16*)cos_t, (const bf16*)sin_t, rows, 1, H, D, ld, 0, nullptr, seg, nullptr);
    B200_CHECK_LAUNCH("rope_seg");
    return B200_OK;
}

extern "C" int b200_rope_qk_ragged(void* qkv, const void* cos_t, const void* sin_t, int rows, int S, int H, int D, int ld,
                                   int pos0, const int* pos0_dev, const int* row_off, cudaStream_t stream) {
    B200_CHECK_ARG(D % 16 == 0 && H % D == 0 && ld % 8 == 0, "rope_ragged: head_dim must be a multiple of 16");
    B200_CHECK_ARG(S >= 1 && row_off != nullptr, "rope_ragged: S >= 1 and row_off required");
    if (rows == 0) return B200_OK;
    rope_kernel<false, true><<<rows, ROW_THREADS, 0, stream>>>((bf16*)qkv, (const bf16*)cos_t, (const bf16*)sin_t, rows, S, H,
                                                              D, ld, pos0, pos0_dev, nullptr, row_off);
    B200_CHECK_LAUNCH("rope_ragged");
    return B200_OK;
}

extern "C" int b200_swiglu_fwd(const void* gu, void* act, long long rows, int I, cudaStream_t stream) {
    B200_CHECK_ARG(I % 8 == 0, "swiglu: intermediate size must be a multiple of 8");
    if (rows == 0) return B200_OK;
    swiglu_fwd_kernel<<<grid_for((size_t)rows * (I / 8), 256), 256, 0, stream>>>((const bf16*)gu, (bf16*)act, rows, I);
    B200_CHECK_LAUNCH("swiglu_fwd");
    return B200_OK;
}

extern "C" int b200_scale_bf16(const void* x, void* y, long long n, float s, cudaStream_t stream) {
    B200_CHECK_ARG(n >= 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, "scale: operands must be 16-byte aligned");
    if (n == 0) return B200_OK;
    scale_bf16_kernel<<<grid_for((size_t)n / 8 + 1, 256), 256, 0, stream>>>((const bf16*)x, (bf16*)y, (size_t)n, s);
    B200_CHECK_LAUNCH("scale_bf16");
    return B200_OK;
}

extern "C" int b200_swiglu_bwd(const void* gu, const void* dact, void* dgu, long long rows, int I, cudaStream_t stream) {
    B200_CHECK_ARG(I % 8 == 0, "swiglu: intermediate size must be a multiple of 8");
    if (rows == 0) return B200_OK;
    swiglu_bwd_kernel<<<grid_for((size_t)rows * (I / 8), 256), 256, 0, stream>>>((const bf16*)gu, (const bf16*)dact,
                                                                                 (bf16*)dgu, rows, I);
    B200_CHECK_LAUNCH("swiglu_bwd");
    return B200_OK;
}
