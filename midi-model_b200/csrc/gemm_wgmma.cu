// bf16 GEMM on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers, operands staged by TMA into
// 128B-swizzled shared memory), persistent, warp-specialised:
//   warps 0..7 : two consumer warpgroups; warpgroup g owns rows [64g, 64g + 64) of the 128-row tile, issues its
//                wgmma chain and runs the fused epilogue straight from its accumulator registers
//   warp 8     : TMA producer (one elected lane)
// D[M,N] = A . B^T with fp32 accumulation.  Each operand is either "K-major"
// (row-major [rows, K], what nn.Linear's forward needs: hf modeling_llama.py:177-184,
// 238-264) or "MN-major" (stored [K, rows]); the latter serves dgrad (B = W as stored)
// and wgrad (A = dY, B = X as stored) without any transposed copies (wgmma's transpose bits).
// Epilogues: bf16 store; bf16 store + residual (two roundings, like `x + o_proj(..)`
// in hf :325/:331); fp32 split-K partials reduced by splitk_reduce_kernel.
#include <math.h>

#include "hopper.cuh"
#include "rope.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int MMA_K = 16;
constexpr int CONSUMERS = 2;                            // consumer warpgroups (64 rows each)
constexpr int NUM_THREADS = CONSUMERS * 128 + 32;       // + the producer warp
constexpr int EPI_BOX_BYTES = 64 * 64 * 2;              // one 64-row x 64-column bf16 box of the TMA store

enum { EPI_STORE = 0, EPI_RESIDUAL = 1, EPI_PARTIAL_F32 = 2, EPI_ROPE = 3, EPI_SWIGLU = 4 };

// EPI_ROPE: rotary embedding applied to columns [0, cols) (the q and k thirds of a packed QKV row) in heads of D columns;
// row r sits at position r % S, or at its in-segment position with a segment table
struct RopeOperands { const bf16 *cos, *sin; const int* seg; int S, D, cols; };
// EPI_SWIGLU: B = [gate | up] weight rows; tile n covers gate rows [128n, 128n+128) and up rows [I + 128n, ...), and
// act[M, I] (pitch ld_act) is written besides gate|up
struct SwigluOperands { bf16* act; int I, ld_act; };

// The epilogue a GEMM call asks for: EPI_STORE (plain, residual or split-K, as its other arguments say), EPI_ROPE or
// EPI_SWIGLU, with the operands of the last two
struct Epilogue { int kind = EPI_STORE; RopeOperands rope = {}; SwigluOperands swiglu = {}; };

struct GemmParams {
    bf16* C;
    const bf16* R;
    float* ws;
    int M, N, K;
    int ldc, ldr;
    int epilogue;
    int splits, kb_per_split, num_kb;
    // tail split: the tiles of the last, partial wave (index >= tail_tile0) are cut into tail_splits K-slices whose fp32
    // partials go to tail_ws[tile - tail_tile0][slice][128][BLOCK_N] and are summed by tail_reduce_kernel
    int tail_tile0, tail_splits, tail_kb, total_items;
    float* tail_ws;
    int m_tiles, n_tiles;
    RopeOperands rope;
    SwigluOperands swiglu;
};

using namespace hopper;

template <int BLOCK_N>
struct SmemLayout {
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB
    static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;   // 16 / 32 KB
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (BLOCK_N == 256) ? 4 : 6;   // 192 KB of operand stages either way
    // bf16 epilogue staging: two 64 x 64 boxes (8 KB, 1024-byte aligned for the 128B swizzle) per consumer warpgroup
    static constexpr int EPI_BYTES = CONSUMERS * 2 * EPI_BOX_BYTES;
    static constexpr int BAR_BYTES = 256;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + EPI_BYTES + BAR_BYTES + 1024;   // +1024 for manual alignment
    static_assert(TOTAL <= 227 * 1024, "shared memory budget of an sm_90 CTA");
};

struct WorkItem {
    int m_blk, n_blk, kb0, kb1, split;
    int tail;          // -1: regular item; otherwise index of the tile inside the tail region
};
__device__ __forceinline__ WorkItem decode_item(const GemmParams& p, int item) {
    WorkItem w;
    const int reg_items = p.tail_tile0 * p.splits;
    int t;
    if (item < reg_items) {
        w.split = item % p.splits;
        t = item / p.splits;
        w.kb0 = w.split * p.kb_per_split;
        w.kb1 = min(w.kb0 + p.kb_per_split, p.num_kb);
        w.tail = -1;
    } else {
        const int idx = item - reg_items;
        w.tail = idx / p.tail_splits;
        w.split = idx % p.tail_splits;
        t = p.tail_tile0 + w.tail;
        w.kb0 = w.split * p.tail_kb;
        w.kb1 = min(w.kb0 + p.tail_kb, p.num_kb);
    }
    w.n_blk = t % p.n_tiles;
    w.m_blk = t / p.n_tiles;
    return w;
}

template <int BLOCK_N, bool TA, bool TB>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (BLOCK_N == 256) wgmma_m64n256k16<TA, TB>(acc, da, db, scale_d);
    else wgmma_m64n128k16<TA, TB>(acc, da, db, scale_d);
}

// Accumulator fragment of wgmma m64nN (fp32): thread (warp w of the warpgroup, lane l) holds, for every 8-column group
// j, acc[4j + h] at row 16w + l/4 + 8 * (h >> 1), column 8j + 2 * (l % 4) + (h & 1).

// RoPE on the fragment, of x = bf16(acc) (the Linear's rounding).  A head of D <= BLOCK_N columns never straddles a
// tile, so both halves of a (d, d + D/2) pair sit in the same thread (groups j and j + HALF8).
template <int BLOCK_N, int HALF8>
__device__ __forceinline__ void rope_fragment(float* acc, const GemmParams& p, int n_blk, int row, int h, int cq) {
    if (row >= p.M) return;
    const int pos = p.rope.seg ? seg_pos(p.rope.seg, row) : row % p.rope.S;
    const int half = HALF8 * 8;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; j++) {
        if ((j / HALF8) & 1) continue;                          // second half of a head: done with its partner
        const int col = n_blk * BLOCK_N + 8 * j + cq;
        if (col >= p.rope.cols) continue;
        const int d = (8 * j) % half + cq;
        const float2 cc = __bfloat1622float2(*reinterpret_cast<const bf162*>(p.rope.cos + (size_t)pos * half + d));
        const float2 ss = __bfloat1622float2(*reinterpret_cast<const bf162*>(p.rope.sin + (size_t)pos * half + d));
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const float c = e ? cc.y : cc.x, s = e ? ss.y : ss.x;
            const float x1 = bf16_round(acc[4 * j + 2 * h + e]);
            const float x2 = bf16_round(acc[4 * (j + HALF8) + 2 * h + e]);
            acc[4 * j + 2 * h + e] = rope_fwd_elem(x1, x2, c, s, false);
            acc[4 * (j + HALF8) + 2 * h + e] = rope_fwd_elem(x2, x1, c, s, true);
        }
    }
}

// One 64 x 64 bf16 box of a warpgroup's output, staged in shared memory and stored by TMA at (col, row0) of `tm`.
// value(jj, h, r) is the thread's packed column pair of 8-column group jj of the box in fragment row half h; r is the
// matching packed pair of the residual `res` (pitch ldr, read only inside rows < M and columns < N), 0 without one.
// The warpgroup alternates between its two staging slots (`boxes` counts the boxes it has issued).  Slot layout = the
// store map's 128B swizzle: row r at byte 128 r, 16-byte chunk c at chunk c ^ (r % 8).  One (jj, h) write of a warp
// covers 8 rows with r % 8 = lane / 4, so 8 distinct chunks, each written by 4 lanes in its 4 banks: all 32 banks once,
// no conflicts.  Before the barrier the elected thread waits until the previous box's store has read its slot, so after
// the barrier the other slot (the next box's) is free; this box's own slot was freed the same way one box earlier.
template <typename F>
__device__ __forceinline__ void store_box(uint8_t* staging, uint32_t& boxes, const CUtensorMap* tm, int col, int row0,
                                          int wg, int r_lo, int lane, bool elected, const bf16* res, int ldr, int M, int N,
                                          F value) {
    uint32_t rv[2][8];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int row = row0 + r_lo + 8 * h;
        const bf16* rp = res + (size_t)row * ldr + col + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 8; jj++)   // all of the box's residual loads in flight before the first shared store
            rv[h][jj] = (res != nullptr && row < M && col + 8 * jj < N) ? *reinterpret_cast<const uint32_t*>(rp + 8 * jj) : 0u;
    }
    uint8_t* slot = staging + (boxes & 1) * EPI_BOX_BYTES;
    // the slot is 1024-byte aligned and r_lo % 8 = lane / 4, so chunk jj ^ (r % 8) of row r is at address ^ (jj << 4)
    const uint32_t s0 = smem_u32(slot) + r_lo * 128 + ((lane >> 2) << 4) + 4 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll
        for (int jj = 0; jj < 8; jj++) st_shared_u32((s0 + h * 8 * 128) ^ (jj << 4), value(jj, h, rv[h][jj]));
    }
    fence_proxy_async_smem();
    if (elected) bulk_wait_read<0>();
    named_bar_sync(1 + wg, 128);
    if (elected) {
        tma_store_2d(tm, slot, col, row0);
        bulk_commit();
    }
    boxes++;
}

template <int BLOCK_N, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAct, const GemmParams p) {
    using L = SmemLayout<BLOCK_N>;
    B200_PDL_TRIGGER();
    constexpr int STAGES = L::STAGES;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES + L::EPI_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == CONSUMERS * 4 && lane == 0) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        if (p.epilogue != EPI_PARTIAL_F32) prefetch_tmap(&tmC);
        if (p.epilogue == EPI_SWIGLU) prefetch_tmap(&tmAct);
        for (int s = 0; s < STAGES; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONSUMERS * 4); // one arrival per consumer warp, each after its own wait
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // everything above may have run under the previous kernel's tail (PDL); from here on this kernel reads and writes
    // global memory
    B200_PDL_WAIT();

    const int total_items = p.total_items;

    if (warp == CONSUMERS * 4) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
                const WorkItem wi = decode_item(p, item);
                for (int kb = wi.kb0; kb < wi.kb1; kb++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sA = smem + stage * L::STAGE_BYTES;
                    uint8_t* sB = sA + L::A_BYTES;
                    mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                    if (!A_MN) {
                        tma_load_2d(sA, &tmA, &full_bar[stage], kb * BLOCK_K, wi.m_blk * BLOCK_M);
                    } else {
#pragma unroll
                        for (int c = 0; c < BLOCK_M / 64; c++)
                            tma_load_2d(sA + c * (BLOCK_K * 128), &tmA, &full_bar[stage], wi.m_blk * BLOCK_M + c * 64, kb * BLOCK_K);
                    }
                    if (!B_MN) {
                        if (BLOCK_N == 256 && p.epilogue == EPI_SWIGLU) {   // gate half | up half (tensor map box = 128 rows)
                            tma_load_2d(sB, &tmB, &full_bar[stage], kb * BLOCK_K, wi.n_blk * 128);
                            tma_load_2d(sB + 128 * BLOCK_K * 2, &tmB, &full_bar[stage], kb * BLOCK_K, p.swiglu.I + wi.n_blk * 128);
                        } else {
                            tma_load_2d(sB, &tmB, &full_bar[stage], kb * BLOCK_K, wi.n_blk * BLOCK_N);
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < BLOCK_N / 64; c++)
                            tma_load_2d(sB + c * (BLOCK_K * 128), &tmB, &full_bar[stage], wi.n_blk * BLOCK_N + c * 64, kb * BLOCK_K);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    const int wg = warp >> 2;                   // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
    const int wr = warp & 3;                    // warp inside the warpgroup: rows 16 wr .. 16 wr + 15 of those
    const int cq = 2 * (lane & 3);              // first of the thread's two columns inside each 8-column group
    const bool signal = lane == 0;
    // A: rows of this warpgroup start 64 rows = 8 KB into the stage either way (K-major: 64 rows x 128 B; MN-major:
    // the second 64-row TMA box).  K-major operands: SBO = 1024 B between 8-row groups, K step = 32 B; MN-major:
    // LBO = 8 KB between 64-element MN boxes, SBO = 1024 B between 8-deep K groups, K step = 16 rows x 128 B.
    const uint32_t a_off = wg * (64 * 128);
    uint8_t* staging = smem + STAGES * L::STAGE_BYTES + wg * (2 * EPI_BOX_BYTES);
    const bool elected = (threadIdx.x & 127) == 0;   // issues and waits for this warpgroup's TMA stores
    const int r_lo = wr * 16 + (lane >> 2);          // the thread's first fragment row inside the warpgroup's 64
    uint32_t boxes = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BLOCK_N / 2];
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        const WorkItem wi = decode_item(p, item);
        int prev = -1;
        for (int kb = wi.kb0; kb < wi.kb1; kb++) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sA = smem_u32(smem + stage * L::STAGE_BYTES) + a_off;
            const uint32_t sB = smem_u32(smem + stage * L::STAGE_BYTES) + L::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / MMA_K; k++) {
                const uint64_t da = A_MN ? make_smem_desc(sA + k * (MMA_K * 128), BLOCK_K * 128, 1024)
                                         : make_smem_desc(sA + k * (MMA_K * 2), 16, 1024);
                const uint64_t db = B_MN ? make_smem_desc(sB + k * (MMA_K * 128), BLOCK_K * 128, 1024)
                                         : make_smem_desc(sB + k * (MMA_K * 2), 16, 1024);
                wgmma_tile<BLOCK_N, A_MN, B_MN>(acc, da, db, (kb > wi.kb0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            // keep this k-block's MMAs in flight; the previous block's have retired, so its stage can be refilled
            wgmma_wait<1>();
            if (prev >= 0 && signal) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        if (prev >= 0 && signal) mbar_arrive(&empty_bar[prev]);

        // ---- epilogue from the accumulator registers
        if (wi.tail >= 0 || p.epilogue == EPI_PARTIAL_F32) {
            // fp32 partials, stored straight from the fragment
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r_t = wg * 64 + r_lo + 8 * h;          // row inside the tile
                if (wi.tail >= 0) {
                    // K-slice of a tail tile: tile-local layout [128][BLOCK_N]
                    float* dst = p.tail_ws + ((size_t)(wi.tail * p.tail_splits + wi.split) * BLOCK_M + r_t) * BLOCK_N + cq;
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 8; j++)
                        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                    continue;
                }
                const int row = wi.m_blk * BLOCK_M + r_t;
                if (row >= p.M) continue;
                float* dst = p.ws + ((size_t)wi.split * p.M + row) * p.N + wi.n_blk * BLOCK_N + cq;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; j++)
                    if (wi.n_blk * BLOCK_N + 8 * j < p.N)
                        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
            continue;
        }
        // bf16 outputs go through shared memory in 64 x 64 boxes and are stored by TMA, which clips rows >= M and
        // columns >= N (= roundup8 of the caller's N; the columns in between hold zeros: B rows >= N were zero-filled);
        // the warpgroup goes on to its next tile's MMAs while the stores drain
        const int row0 = wi.m_blk * BLOCK_M + wg * 64;
        if (row0 >= p.M) continue;
        if (p.epilogue == EPI_ROPE) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row = row0 + r_lo + 8 * h;
                if (p.rope.D == 64) rope_fragment<BLOCK_N, 4>(acc, p, wi.n_blk, row, h, cq);
                else if (p.rope.D == 128) rope_fragment<BLOCK_N, 8>(acc, p, wi.n_blk, row, h, cq);
                else rope_fragment<BLOCK_N, 16>(acc, p, wi.n_blk, row, h, cq);
            }
        }
        if (BLOCK_N == 256 && p.epilogue == EPI_SWIGLU) {
            // gate|up projection with SwiGLU fused (hf modeling_llama.py:183): accumulator columns [0,128) are gate
            // features, [128,256) the matching up features.  g, u = bf16(acc) are stored (backward needs them) and
            // act = bf16(bf16(silu(g)) * u) -- same rounding points as the stand-alone kernel.
            const int f0 = wi.n_blk * 128;
#pragma unroll
            for (int q = 0; q < 2; q++) {
                store_box(staging, boxes, &tmC, f0 + 64 * q, row0, wg, r_lo, lane, elected, nullptr, 0, 0, 0,
                          [&](int jj, int h, uint32_t) {
                    const int j = 8 * q + jj;
                    return pack2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                });
            }
#pragma unroll
            for (int q = 0; q < 2; q++) {
                store_box(staging, boxes, &tmC, p.swiglu.I + f0 + 64 * q, row0, wg, r_lo, lane, elected, nullptr, 0, 0, 0,
                          [&](int jj, int h, uint32_t) {
                    const int j = 16 + 8 * q + jj;
                    return pack2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                });
            }
#pragma unroll
            for (int q = 0; q < 2; q++) {
                store_box(staging, boxes, &tmAct, f0 + 64 * q, row0, wg, r_lo, lane, elected, nullptr, 0, 0, 0,
                          [&](int jj, int h, uint32_t) {
                    const int j = 8 * q + jj;
                    const float g0 = bf16_round(acc[4 * j + 2 * h]), g1 = bf16_round(acc[4 * j + 2 * h + 1]);
                    const float u0 = bf16_round(acc[4 * (j + 16) + 2 * h]), u1 = bf16_round(acc[4 * (j + 16) + 2 * h + 1]);
                    return pack2(bf16_round(silu_f(g0)) * u0, bf16_round(silu_f(g1)) * u1);
                });
            }
        } else {
            // plain / residual / RoPE'd bf16 store
            const bool residual = p.epilogue == EPI_RESIDUAL;
#pragma unroll
            for (int b = 0; b < BLOCK_N / 64; b++) {
                const int col = wi.n_blk * BLOCK_N + 64 * b;
                if (col >= p.N) break;
                store_box(staging, boxes, &tmC, col, row0, wg, r_lo, lane, elected, residual ? p.R : nullptr, p.ldr, p.M,
                          p.N, [&](int jj, int h, uint32_t r) {
                    const int j = 8 * b + jj;
                    float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                    if (residual) {
                        const float2 rr = __bfloat1622float2(*reinterpret_cast<const bf162*>(&r));
                        f0 = bf16_round(f0) + rr.x;
                        f1 = bf16_round(f1) + rr.y;
                    }
                    return pack2(f0, f1);
                });
            }
        }
    }
    // the staging slots must stay untouched until the last stores have read them; the CTA exits after they completed
    if (elected) bulk_wait_all();
}

__global__ void splitk_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ out, size_t n, int splits,
                                     int accumulate) {
    size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const size_t stride = (size_t)gridDim.x * blockDim.x * 4;
    for (; i < n; i += stride) {
        float4 a = *reinterpret_cast<const float4*>(ws + i);
        for (int s = 1; s < splits; s++) {
            float4 b = *reinterpret_cast<const float4*>(ws + (size_t)s * n + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        bf162* o = reinterpret_cast<bf162*>(out + i);
        if (accumulate) {   // grad accumulation across micro-batches: bf16 += bf16(new), like autograd's AccumulateGrad
            float2 o0 = __bfloat1622float2(o[0]), o1 = __bfloat1622float2(o[1]);
            a.x = bf16_round(a.x) + o0.x; a.y = bf16_round(a.y) + o0.y;
            a.z = bf16_round(a.z) + o1.x; a.w = bf16_round(a.w) + o1.y;
        }
        o[0] = __floats2bfloat162_rn(a.x, a.y);
        o[1] = __floats2bfloat162_rn(a.z, a.w);
    }
}

// sums the K-slices of the tail tiles and writes bf16 into C (rows < M, columns < N, N a multiple of 8)
__global__ void tail_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ C, int M, int N, int ldc, int n_tiles,
                                   int tail_tile0, int n_tail, int splits, int block_n) {
    const int per_tile = BLOCK_M * block_n / 8;                 // 8-column groups per tile
    const long long total = (long long)n_tail * per_tile;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int tt = (int)(i / per_tile), e = (int)(i % per_tile);
        const int r = e / (block_n / 8), c8 = e % (block_n / 8);
        const int t = tail_tile0 + tt;
        const int row = (t / n_tiles) * BLOCK_M + r, col = (t % n_tiles) * block_n + c8 * 8;
        if (row >= M || col >= N) continue;
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int s = 0; s < splits; s++) {
            const float* src = ws + ((size_t)(tt * splits + s) * BLOCK_M + r) * block_n + c8 * 8;
            const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
            acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
            acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
        }
        *reinterpret_cast<uint4*>(C + (size_t)row * ldc + col) = pack8(acc);
    }
}

template <int BLOCK_N, bool A_MN, bool B_MN>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmAct,
           const GemmParams& p, cudaStream_t stream) {
    using L = SmemLayout<BLOCK_N>;
    auto kern = gemm_wgmma_kernel<BLOCK_N, A_MN, B_MN>;
    static bool configured = false;
    if (!configured) {
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL), "gemm smem attr");
        configured = true;
    }
    const int items = p.total_items;
    static int pdl = -1;
    if (pdl < 0) {
        // B200_PDL=1: programmatic dependent launch of the GEMMs (off by default).
        const char* e = getenv("B200_PDL");
        pdl = (e && e[0] == '1') ? 1 : 0;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = L::TOTAL;
    cfg.stream = stream;
    cfg.gridDim = dim3(items < b200_num_sms() ? items : b200_num_sms());
    cudaLaunchAttribute attr[1];
    int n_attr = 0;
    if (pdl) {
        attr[n_attr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n_attr].val.programmaticStreamSerializationAllowed = 1;
        n_attr++;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n_attr;
    B200_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, tmAct, p), "gemm launch");
    B200_CHECK_LAUNCH("gemm_wgmma");
    return B200_OK;
}

}   // namespace

// ---------------------------------------------------------------------------
// host side: tensor maps through the driver entry point (no -lcuda link dependency)
// ---------------------------------------------------------------------------
namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

// 2-D bf16 tensor map: `inner` contiguous elements, `outer` rows of pitch `ld` elements, 128B swizzle, zero OOB fill.
}   // namespace

int hopper::make_tmap_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                       uint32_t box_outer) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        b200_set_error("gemm: cuTensorMapEncodeTiled entry point unavailable");
        return B200_ERR_CUDA;
    }
    cuuint64_t gdim[2] = {inner, outer};
    cuuint64_t gstride[1] = {ld * 2};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        b200_set_error("gemm: cuTensorMapEncodeTiled failed (%d) ptr=%p inner=%llu outer=%llu ld=%llu", (int)r, ptr,
                       (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld);
        return B200_ERR_CUDA;
    }
    return B200_OK;
}

int hopper::make_tmap_3d(CUtensorMap* tm, const void* ptr, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t row_pitch,
                         uint64_t batch_pitch, uint32_t box_cols, uint32_t box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        b200_set_error("tmap3d: cuTensorMapEncodeTiled entry point unavailable");
        return B200_ERR_CUDA;
    }
    cuuint64_t gdim[3] = {cols, rows, batch};
    cuuint64_t gstride[2] = {row_pitch * 2, batch_pitch * 2};
    cuuint32_t box[3] = {box_cols, box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        b200_set_error("tmap3d: cuTensorMapEncodeTiled failed (%d) ptr=%p cols=%llu rows=%llu batch=%llu pitch=%llu/%llu",
                       (int)r, ptr, (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)batch,
                       (unsigned long long)row_pitch, (unsigned long long)batch_pitch);
        return B200_ERR_CUDA;
    }
    return B200_OK;
}

// ---------------------------------------------------------------------------
// C ABI (declared in include/midi_b200.h)
// ---------------------------------------------------------------------------
// fp32 partials of a call that splits K or accumulates (accumulate with splits == 1 still needs one M x N slice)
extern "C" size_t b200_gemm_workspace_bytes(int M, int N, int splits) {
    return (size_t)(splits > 1 ? splits : 1) * M * N * sizeof(float);
}

// Tail split.  tiles = full * sms + r: the last wave keeps only r of the sms CTAs busy for a whole tile time.  Cutting
// those r tiles into s K-slices makes the tail ceil(r*s/sms)/s tile times long (e.g. 512 tiles on 132 SMs: r = 116,
// s = 2 -> 3.5 instead of 4 waves).  Returns s (1 = leave the tail alone).
static int plan_tail(int tiles, int num_kb, int sms) {
    static int enabled = -1;
    if (enabled < 0) {
        const char* e = getenv("B200_GEMM_TAIL_SPLIT");
        enabled = (e && e[0] == '0') ? 0 : 1;
    }
    const int full = tiles / sms, r = tiles % sms;
    // long K only (the fp32 partial round trip and the extra reduce launch must be small next to the half wave saved),
    // 2-way only
    if (!enabled || r == 0 || full == 0 || full > 8 || num_kb < 96) return 1;
    const double cost = (double)((r * 2 + sms - 1) / sms) / 2 + 0.06;
    return cost < 0.75 ? 2 : 1;
}

// bytes of fp32 workspace b200_gemm_bf16 can use to split the tiles of the last partial wave along K (0: no tail split
// for this shape).  Optional: without the workspace the GEMM runs unsplit.
extern "C" size_t b200_gemm_tail_workspace_bytes(int M, int N, int K, int block_n) {
    if (block_n != 128 && block_n != 256) return 0;
    const int tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + block_n - 1) / block_n);
    const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    const int sms = b200_num_sms();
    const int s = plan_tail(tiles, num_kb, sms);
    return s > 1 ? (size_t)(tiles % sms) * s * BLOCK_M * block_n * sizeof(float) : 0;
}

// Tile / split-K planner.  Work items = tiles(block_n) x splits run persistently on `sms` CTAs, so the cost is
// (waves of items) x (k-blocks per item) in MMA clocks, plus pipeline fill, the exposed last epilogue and, for
// splits > 1, the fp32 partial round trip.  Picks the cheapest (block_n, splits): this is what removes the
// wave-quantisation loss of the small-output wgrad problems (e.g. 192 tiles on 132 SMs -> 2 splits, 2.9 waves).
static double plan_cost(int M, int N, int K, int block_n, int s, int sms) {
    const double tiles = (double)((M + BLOCK_M - 1) / BLOCK_M) * ((N + block_n - 1) / block_n);
    const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    const int kb_per = (num_kb + s - 1) / s;
    const int s_eff = (num_kb + kb_per - 1) / kb_per;
    const double items = tiles * s_eff;
    const double waves = ceil(items / sms);
    // 4 wgmma steps of 128 x block_n x 16 per k-block.  A 128-wide tile reads more shared-memory operand bytes per FLOP
    // than a 256-wide one (each warpgroup re-reads its A rows for half the columns), hence its higher cost per column.
    const double kb_clk = 2.0 * block_n * (block_n == 128 ? 1.25 : 1.0);
    const double tile_ovh = 150.0 + (s_eff > 1 ? 1.0 : 0.5) * block_n * 6.0;   // accumulator hand-over + epilogue pressure
    double c = waves * (kb_per * kb_clk + tile_ovh) + 2500.0;   // + fill and exposed tail epilogue
    if (s_eff > 1) c += ((double)s_eff * M * N * 8.0 + (double)M * N * 2.0) / 5000.0 + 4000.0;   // bytes / (B/clk, mostly L2) + launch
    return c;
}

extern "C" int b200_gemm_plan(int M, int N, int K, int allow_split, int* block_n_out, int* splits_out) {
    const int sms = b200_num_sms();
    double best = 1e300;
    int bb = 128, bs = 1;
    for (int bn = 128; bn <= 256; bn += 128) {
        if (bn == 256 && N < 256) continue;
        const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
        const int smax = allow_split ? (num_kb / 8 > 16 ? 16 : (num_kb / 8 > 0 ? num_kb / 8 : 1)) : 1;
        for (int s = 1; s <= smax; s++) {
            const double c = plan_cost(M, N, K, bn, s, sms);
            if (c < best) { best = c; bb = bn; bs = s; }
        }
    }
    *block_n_out = bb;
    *splits_out = bs;
    return B200_OK;
}

// legacy helper (kept for ABI stability): split factor for a fixed block_n
extern "C" int b200_gemm_suggest_splits(int M, int N, int K, int block_n) {
    const int sms = b200_num_sms();
    const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    const int smax = num_kb / 8 > 16 ? 16 : (num_kb / 8 > 0 ? num_kb / 8 : 1);
    double best = 1e300;
    int bs = 1;
    for (int s = 1; s <= smax; s++) {
        const double c = plan_cost(M, N, K, block_n, s, sms);
        if (c < best) { best = c; bs = s; }
    }
    return bs;
}

static int gemm_impl(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda, int ldb, int ldc,
                     int ldr, int a_mn_major, int b_mn_major, int accumulate, int block_n, int splits, void* workspace,
                     size_t workspace_bytes, const Epilogue& epi, cudaStream_t stream);

extern "C" int b200_gemm_bf16(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda, int ldb,
                              int ldc, int ldr, int a_mn_major, int b_mn_major, int accumulate, int block_n, int splits,
                              void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    return gemm_impl(A, B, C, R, M, N, K, lda, ldb, ldc, ldr, a_mn_major, b_mn_major, accumulate, block_n, splits, workspace,
                     workspace_bytes, Epilogue{}, stream);
}

// Fused QKV projection + RoPE: C[M,N] = rope(A . B^T) with both operands K-major; rows are positions r % S of their
// sequence, columns [0, rope_cols) are heads of width head_dim that get rotated, the rest (v) is stored as is.
extern "C" int b200_gemm_bf16_rope(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                                   const void* rope_cos, const void* rope_sin, int S, int head_dim, int rope_cols,
                                   cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == 64 || head_dim == 128 || head_dim == 256, "gemm_rope: head_dim %d unsupported", head_dim);
    B200_CHECK_ARG(N % 256 == 0 && rope_cols % 256 == 0, "gemm_rope: N and rope_cols must be multiples of 256");
    B200_CHECK_ARG(S > 0 && rope_cos && rope_sin, "gemm_rope: missing tables");
    const Epilogue epi{EPI_ROPE, {(const bf16*)rope_cos, (const bf16*)rope_sin, nullptr, S, head_dim, rope_cols}};
    return gemm_impl(A, B, C, nullptr, M, N, K, lda, ldb, ldc, 0, 0, 0, 0, 256, 1, nullptr, 0, epi, stream);
}

// The same with in-segment positions (segments of whole 64-row tiles, rope.cuh).
extern "C" int b200_gemm_bf16_rope_seg(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                                       const void* rope_cos, const void* rope_sin, const int* seg, int head_dim,
                                       int rope_cols, cudaStream_t stream) {
    B200_CHECK_ARG(head_dim == 64 || head_dim == 128 || head_dim == 256, "gemm_rope_seg: head_dim %d unsupported", head_dim);
    B200_CHECK_ARG(N % 256 == 0 && rope_cols % 256 == 0, "gemm_rope_seg: N and rope_cols must be multiples of 256");
    B200_CHECK_ARG(M % SEG_TILE == 0 && seg && rope_cos && rope_sin, "gemm_rope_seg: M (%d) must be whole 64-row tiles; "
                   "tables required", M);
    const Epilogue epi{EPI_ROPE, {(const bf16*)rope_cos, (const bf16*)rope_sin, seg, 1, head_dim, rope_cols}};
    return gemm_impl(A, B, C, nullptr, M, N, K, lda, ldb, ldc, 0, 0, 0, 0, 256, 1, nullptr, 0, epi, stream);
}

// Fused gate|up projection + SwiGLU: gu[M, 2I] = A . Wgu^T (stored, the backward pass needs g and u) and
// act[M, I] = bf16(bf16(silu(g)) * u) written by the same epilogue.  Wgu = [gate rows | up rows], K-major operands.
extern "C" int b200_gemm_bf16_swiglu(const void* A, const void* Wgu, void* gu, void* act, int M, int I, int K, int lda,
                                     int ldw, int ld_gu, int ld_act, cudaStream_t stream) {
    B200_CHECK_ARG(I % 128 == 0, "gemm_swiglu: intermediate size %d must be a multiple of 128", I);
    B200_CHECK_ARG(ld_act % 8 == 0 && (uintptr_t)act % 16 == 0, "gemm_swiglu: act must be 16-byte aligned");
    const Epilogue epi{EPI_SWIGLU, {}, {(bf16*)act, I, ld_act}};
    return gemm_impl(A, Wgu, gu, nullptr, M, 2 * I, K, lda, ldw, ld_gu, 0, 0, 0, 0, 256, 1, nullptr, 0, epi, stream);
}

static int gemm_impl(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda, int ldb, int ldc,
                     int ldr, int a_mn_major, int b_mn_major, int accumulate, int block_n, int splits, void* workspace,
                     size_t workspace_bytes, const Epilogue& epi, cudaStream_t stream) {
    const bool swiglu = epi.kind == EPI_SWIGLU;
    B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
    // N need not be a multiple of 8: B rows >= N are out of bounds for the tensor map (zero-filled), so the
    // epilogue may store whole 16-byte vectors up to roundup8(N) (zeros) as long as the row pitch covers them.
    const int N8 = (N + 7) / 8 * 8;
    B200_CHECK_ARG(ldc % 8 == 0 && ldc >= N8, "gemm: ldc (%d) must be a multiple of 8 and >= roundup8(N=%d)", ldc, N);
    B200_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8 (16-byte TMA strides)");
    B200_CHECK_ARG(((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0) && ((uintptr_t)C % 16 == 0),
                   "gemm: operands must be 16-byte aligned");
    B200_CHECK_ARG(block_n == 128 || block_n == 256, "gemm: block_n must be 128 or 256");
    B200_CHECK_ARG(R == nullptr || (ldr % 8 == 0 && (uintptr_t)R % 16 == 0 && N % 8 == 0),
                   "gemm: residual must be 16-byte aligned and N a multiple of 8");
    if (splits < 1) splits = 1;
    GemmParams p;
    p.C = (bf16*)C;
    p.R = (const bf16*)R;
    p.ws = (float*)workspace;
    p.M = M; p.N = N8; p.K = K;
    p.ldc = ldc; p.ldr = ldr;
    p.num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    if (splits > p.num_kb) splits = p.num_kb;
    p.kb_per_split = (p.num_kb + splits - 1) / splits;
    splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;   // no empty splits
    p.splits = splits;
    p.m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    p.n_tiles = (N + block_n - 1) / block_n;
    if (!swiglu && (splits > 1 || accumulate)) {
        B200_CHECK_ARG(R == nullptr, "gemm: split-K/accumulate cannot be combined with a residual epilogue");
        B200_CHECK_ARG(ldc == N && N % 8 == 0, "gemm: split-K/accumulate output must be contiguous (ldc == N, N %% 8 == 0)");
        const size_t need = (size_t)splits * M * N * sizeof(float);
        B200_CHECK_ARG(workspace != nullptr && workspace_bytes >= need, "gemm: workspace too small (%zu < %zu)",
                       workspace_bytes, need);
        p.epilogue = EPI_PARTIAL_F32;
    } else {
        p.epilogue = R ? EPI_RESIDUAL : EPI_STORE;
    }
    if (epi.kind != EPI_STORE) p.epilogue = epi.kind;
    p.rope = epi.rope;
    p.swiglu = epi.swiglu;
    if (swiglu) p.n_tiles = p.swiglu.I / 128;   // one tile = 128 gate + 128 up features

    CUtensorMap tmA, tmB;
    int rc;
    // tail split (plain bf16 store, no split-K, no accumulate) when the caller provided the optional workspace
    p.total_items = p.m_tiles * p.n_tiles * p.splits;
    p.tail_tile0 = p.m_tiles * p.n_tiles;
    p.tail_splits = 1; p.tail_kb = p.num_kb; p.tail_ws = nullptr;
    int n_tail = 0;
    if (p.epilogue == EPI_STORE && p.splits == 1 && !accumulate && workspace != nullptr) {
        const int tiles = p.m_tiles * p.n_tiles, sms = b200_num_sms();
        const int ts = plan_tail(tiles, p.num_kb, sms);
        const size_t need = (size_t)(tiles % sms) * ts * BLOCK_M * block_n * sizeof(float);
        if (ts > 1 && workspace_bytes >= need && ((uintptr_t)workspace % 16 == 0)) {
            n_tail = tiles % sms;
            p.tail_tile0 = tiles - n_tail;
            p.tail_splits = ts;
            p.tail_kb = (p.num_kb + ts - 1) / ts;
            p.tail_splits = (p.num_kb + p.tail_kb - 1) / p.tail_kb;      // no empty slices
            p.tail_ws = (float*)workspace;
            p.total_items = p.tail_tile0 + n_tail * p.tail_splits;
        }
    }
    if (!a_mn_major) rc = hopper::make_tmap_2d(&tmA, A, K, M, lda, BLOCK_K, BLOCK_M);
    else             rc = hopper::make_tmap_2d(&tmA, A, M, K, lda, 64, BLOCK_K);
    if (rc) return rc;
    if (!b_mn_major) rc = hopper::make_tmap_2d(&tmB, B, K, N, ldb, BLOCK_K, swiglu ? 128 : block_n);
    else             rc = hopper::make_tmap_2d(&tmB, B, N, K, ldb, 64, BLOCK_K);
    if (rc) return rc;
    // bf16 outputs: 64 x 64 boxes stored from the epilogue's staging slots (unused maps stay zero)
    CUtensorMap tmC = {}, tmAct = {};
    if (p.epilogue != EPI_PARTIAL_F32) {
        rc = hopper::make_tmap_2d(&tmC, C, N8, M, ldc, 64, 64);
        if (rc) return rc;
    }
    if (swiglu) {
        rc = hopper::make_tmap_2d(&tmAct, p.swiglu.act, p.swiglu.I, M, p.swiglu.ld_act, 64, 64);
        if (rc) return rc;
    }

#define B200_DISPATCH(BN)                                                                                  \
    do {                                                                                                   \
        if (!a_mn_major && !b_mn_major) rc = launch<BN, false, false>(tmA, tmB, tmC, tmAct, p, stream);    \
        else if (!a_mn_major && b_mn_major) rc = launch<BN, false, true>(tmA, tmB, tmC, tmAct, p, stream); \
        else if (a_mn_major && b_mn_major) rc = launch<BN, true, true>(tmA, tmB, tmC, tmAct, p, stream);   \
        else rc = launch<BN, true, false>(tmA, tmB, tmC, tmAct, p, stream);                                \
    } while (0)
    if (block_n == 256) B200_DISPATCH(256);
    else B200_DISPATCH(128);
#undef B200_DISPATCH
    if (rc) return rc;

    if (n_tail > 0) {
        const long long groups = (long long)n_tail * BLOCK_M * block_n / 8;
        int blocks = (int)((groups + 255) / 256);
        if (blocks > b200_num_sms() * 8) blocks = b200_num_sms() * 8;
        tail_reduce_kernel<<<blocks, 256, 0, stream>>>(p.tail_ws, p.C, M, N8, ldc, p.n_tiles, p.tail_tile0, n_tail, p.tail_splits, block_n);
        B200_CHECK_LAUNCH("gemm_tail_reduce");
    }
    if (p.epilogue == EPI_PARTIAL_F32) {
        const size_t n = (size_t)M * N;
        int blocks = (int)((n / 4 + 255) / 256);
        if (blocks > b200_num_sms() * 8) blocks = b200_num_sms() * 8;
        splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(p.ws, p.C, n, splits, accumulate);
        B200_CHECK_LAUNCH("splitk_reduce");
    }
    return B200_OK;
}
