// Persistent generate kernel: ONE cooperative launch runs whole generated events of MIDIModel.generate
// (midi_model.py:192-248) -- the event-level decode step over the paged KV cache, up to 8 token-level decode steps with
// grammar-masked sampling, and the commit of the event -- on one CTA per SM, with a grid-wide barrier between the
// dependent phases instead of a kernel boundary.  Per layer: norm+QKV | RoPE+append+attention | (combine) |
// o_proj+residual | norm+gate/up+SwiGLU | down+residual; per token: ... | final norm+lm_head | sample.
//
// Why: at batch 1 a decode step moves < 0.5 GB (~150 us at H100 HBM speed) but the launch-per-phase loop needs ~210 graph nodes
// per event, each a launch with its own fixed cost.  Here a phase boundary is a grid barrier instead, and each
// warp issues the loads of its first weight rows of the NEXT phase before it waits at the barrier (weights do not depend
// on the previous phase), so the HBM latency of every phase hides behind the barrier.
//
// A grid barrier waits for the issuing SM's outstanding loads (tools/micro/gridbar_bench.cu measures its cost), so a
// phase boundary costs more than one L2 round trip.  The phases stay inlined: shared non-inlined routines put their
// argument structs in local memory.
//
// Arithmetic and rounding points are those of the launch-per-phase kernels in decode.cu (same per-row accumulation
// order in the projections; attention differs only in how the context is cut into chunks).
#include <cooperative_groups.h>
#include <type_traits>

#include "common.cuh"
#include "rope.cuh"
#include "sampler.cuh"
#include "../../include/midi_b200.h"

namespace {

constexpr int PD_THREADS = 512;
constexpr int PD_WARPS = PD_THREADS / 32;
constexpr int PD_MAXC = 160;             // attention chunks per (row, head)
constexpr int PD_T = 8;                  // tokens per event

struct DD {                              // b200_decode_desc with typed pointers
    const long long *outer_w, *inner_w;
    int n_outer, n_inner;
    const bf16 *outer_norm, *inner_norm, *lm_head, *emb_outer, *emb_inner;
    int H, I_outer, I_inner, nh_outer, nh_inner, V, pitch;
    float eps;
    const long long* kv_outer;
    const int* block_table;
    int max_pages, page;
    const bf16 *cos_outer, *sin_outer, *cos_inner, *sin_inner;
    int* pos;
    long long *ev_in, *seq;
    int max_len;
    unsigned long long* rng_state;
    const unsigned char* dense_mask;
    const int* lut;
    int n_event_types, eos_id, pad_id;
    float temp, top_p;
    int top_k, batch;
    unsigned long long* prof;            // optional: per-phase clock64 totals of CTA 0 (tuning hook)
};

struct PD {                              // kernel parameters (device pointers resolved on the host)
    DD d;
    // workspace carve-up
    unsigned int* bar;
    bf16 *x, *h, *x2, *h2, *qkv, *attn, *act, *logits;
    long long* ev_t;                     // [8][B]
    float* partial;                      // [B*nh][PD_MAXC][D+2]
    bf16 *k2, *v2;                       // [n_inner][B][8][H]
    int n_events;
    int k_max;
};
// parameters of the ragged kernel (b200_decode_events_ragged): PD plus the per-row position offsets.  A derived struct
// rather than a new PD field, so that the kernel without RAGGED keeps its parameter block (and its stack copy of it).
struct PDRagged : PD {
    const int* row_off;                  // [B]: row b's position is pos + row_off[b] <= pos
};
// parameters of the request-queue kernel (b200_decode_events_queue): the ragged ones plus each row's budget and state
struct PDQueue : PDRagged {
    const int* row_end;                  // [B]: seq index of row b's last allowed event
    int* row_last;                       // [B]: -1 while row b is live, else the seq index of its last event (-2: empty)
    int exit_on_done;                    // leave after the event in which a row finished
};
// parameters of the per-request queue kernel (b200_decode_events_queue_rows): the queue ones plus each row's sampling
// settings and RNG key; row b's new event j = pos + row_off[b] - row_first[b] draws hash(row_seed[b], 8 j + t, 0)
struct PDRows : PDQueue {
    const float *row_temp, *row_top_p;   // [B]
    const int* row_top_k;                // [B], 1..128
    const unsigned long long* row_seed;  // [B]
    const int* row_first;                // [B]: seq index of the request's last prompt event
};
// parameters of the streaming queue kernel (b200_decode_events_queue_stream): the per-request ones plus the host mirror of
// the committed events and the host's "leave soon" flag (device pointers of pinned host memory)
struct PDStream : PDRows {
    long long* out_events;               // [B][max_len][8]: each committed event, at its seq index
    int* committed;                      // [B]: seq index of row b's last committed event (release after the event)
    const int* ctl;                      // the host sets it nonzero to end the launch
    int* ctl_seen;                       // workspace word: ctl as CTA 0 read it in this event
};
template <bool RAGGED, bool QUEUE = false, bool ROWS = false, bool STREAM = false>
using PDArg = std::conditional_t<STREAM, PDStream, std::conditional_t<ROWS, PDRows, std::conditional_t<QUEUE, PDQueue,
              std::conditional_t<RAGGED, PDRagged, PD>>>>;

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int ld_acquire_sys_s32(const int* p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_s32(int* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
// weights: read-only for the whole launch.  Event-level weights (403 MB) are streamed once per event -> evict first, so
// that as much as possible of the token-level weights (51 MB, re-read by each of the 8 token steps) stays in the 50 MB L2.
// (L2 eviction priority through a createpolicy cache hint.)
__device__ __forceinline__ unsigned long long l2_policy(bool keep) {
    unsigned long long pol;
    if (keep) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    else asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint4 ldw16(const void* p, unsigned long long pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}

struct GridBar {
    unsigned int* ctr;
    unsigned int target, n;
};
// All CTAs are co-resident (cooperative launch).  CTA barrier; one thread publishes with a release reduction and polls
// with relaxed loads until every CTA of this generation has arrived; CTA barrier.  No acquire fence is needed after the
// poll: every cross-CTA datum of this kernel is read with ld.global.cg (L2, where the release made it visible) and only
// after the closing bar.sync, and a gpu-scope acquire would cost an L1 invalidation (CCTL.IVALL) per poll.  The polling
// thread belongs to warp 0, which never has prefetch loads in flight (a release waits for the issuing thread's own
// outstanding loads).  The spin is bounded: a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void grid_sync(GridBar& gb) {
    __syncthreads();
    gb.target += gb.n;
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(gb.ctr) : "memory");
        unsigned v;
        unsigned spins = 0;
        long long t0 = 0;
        for (;;) {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(gb.ctr) : "memory");
            if (v >= gb.target) break;
            if ((++spins & 1023u) == 0) {
                if (t0 == 0) t0 = clock64();
                else if (clock64() - t0 > 4000000000LL) {
                    printf("b200: decode grid barrier timeout (block %d, target %u, counter %u)\n", blockIdx.x, gb.target, v);
                    __trap();
                }
            }
        }
    }
    __syncthreads();
}

// tuning hook: phase id -> cycles spent by CTA 0 between the barrier that opened the phase and the one that closed it
enum { PH_QKV_O, PH_ATT_O, PH_CMB_O, PH_OPROJ_O, PH_GU_O, PH_DOWN_O, PH_QKV_I, PH_ATT_I, PH_OPROJ_I, PH_GU_I, PH_DOWN_I,
       PH_LMHEAD, PH_SAMPLE, PH_COMMIT, PH_COUNT };
struct Prof {
    unsigned long long* buf;
    long long last, last_sub;
    __device__ __forceinline__ void mark(int id) {
        if (buf != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
            const long long t = clock64();
            buf[id] += (unsigned long long)(t - last);
            buf[32 + id] += 1ull;
            last = t;
            last_sub = t;
        }
    }
    // sub-interval k of phase id (0: staging the activations, 1: the phase's own work; the rest is barrier wait)
    __device__ __forceinline__ void sub(int id, int k) {
        if (buf != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
            const long long t = clock64();
            buf[64 + id * 2 + k] += (unsigned long long)(t - last_sub);
            last_sub = t;
        }
    }
};

struct LayerW {
    const bf16 *qkv, *o, *gu, *down, *ln1, *ln2;
};
__device__ __forceinline__ LayerW layer_w(const long long* tab, int l) {
    LayerW w;
    w.qkv = reinterpret_cast<const bf16*>(tab[l * 6 + 0]);
    w.o = reinterpret_cast<const bf16*>(tab[l * 6 + 1]);
    w.gu = reinterpret_cast<const bf16*>(tab[l * 6 + 2]);
    w.down = reinterpret_cast<const bf16*>(tab[l * 6 + 3]);
    w.ln1 = reinterpret_cast<const bf16*>(tab[l * 6 + 4]);
    w.ln2 = reinterpret_cast<const bf16*>(tab[l * 6 + 5]);
    return w;
}

// ---- skinny projection: every warp owns PAIRS of weight rows -------------------------------------------------
struct Pre {
    uint4 w[2][4];                       // first four 16-byte vectors per lane of the warp's first two rows
};
// rows of pair `pi`: (2 pi, 2 pi + 1), or (pi, pi + N_out) for the gate|up projection
template <bool SWIGLU>
__device__ __forceinline__ void pair_rows(int pi, int N_out, int& r0, int& r1, bool& has1) {
    if (SWIGLU) { r0 = pi; r1 = pi + N_out; has1 = true; }
    else { r0 = 2 * pi; r1 = 2 * pi + 1; has1 = r1 < N_out; }
}
template <bool SWIGLU>
__device__ __forceinline__ void prefetch_rows(Pre& pre, const bf16* __restrict__ W, int ldw, int N_out, int gw, int lane, unsigned long long keep) {
    const int n_pairs = SWIGLU ? N_out : (N_out + 1) / 2;
    if (gw >= n_pairs) return;
    int r0, r1;
    bool has1;
    pair_rows<SWIGLU>(gw, N_out, r0, r1, has1);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        pre.w[0][i] = ldw16(W + (size_t)r0 * ldw + (lane + 32 * i) * 8, keep);
        if (has1) pre.w[1][i] = ldw16(W + (size_t)r1 * ldw + (lane + 32 * i) * 8, keep);
    }
}

// y[b][n] = epi(sum_k xs[b][k] W[n][k]) for this warp's row pairs.  xs: shared [B][K] bf16.  K % 256 == 0.
//   plain   : y = bf16(acc)                         (nn.Linear rounding)
//   res     : y = bf16(bf16(acc) + res[b][n])       (hf modeling_llama.py:325/:331)
//   SWIGLU  : y[b][n] = bf16(bf16(silu(g)) * u), g/u = bf16(acc of rows n / n + N_out)   (hf :183)
template <int BM, bool SWIGLU>
__device__ __forceinline__ void gemv_pairs(const bf16* xs, int K, const bf16* __restrict__ W, int ldw, int N_out, int B,
                                           const bf16* res, int ldr, bf16* y, int ldy, int gw, int ngw, int lane,
                                           const Pre& pre, unsigned long long keep) {
    const int n_pairs = SWIGLU ? N_out : (N_out + 1) / 2;
    const int nblk = K / 256;            // blocks of 32 lanes x 8 elements
    for (int pi = gw; pi < n_pairs; pi += ngw) {
        int r0, r1;
        bool has1;
        pair_rows<SWIGLU>(pi, N_out, r0, r1, has1);
        const bf16* w0p = W + (size_t)r0 * ldw;
        const bf16* w1p = W + (size_t)(has1 ? r1 : r0) * ldw;
        float acc0[BM], acc1[BM];
#pragma unroll
        for (int b = 0; b < BM; b++) { acc0[b] = 0.f; acc1[b] = 0.f; }
        // residual values of this pair (lane b <-> batch row b): requested now, needed only after the reduction
        unsigned short res0 = 0, res1 = 0;
        if (!SWIGLU && res != nullptr && lane < B) {
            res0 = __ldcg(reinterpret_cast<const unsigned short*>(res + (size_t)lane * ldr + r0));
            if (has1) res1 = __ldcg(reinterpret_cast<const unsigned short*>(res + (size_t)lane * ldr + r1));
        }
        const bool first = (pi == gw);
        for (int i0 = 0; i0 < nblk; i0 += 4) {
            uint4 wa[4], wb[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (first && i0 == 0) { wa[i] = pre.w[0][i]; wb[i] = pre.w[1][i]; }
                else {
                    wa[i] = ldw16(w0p + (lane + 32 * (i0 + i)) * 8, keep);
                    wb[i] = ldw16(w1p + (lane + 32 * (i0 + i)) * 8, keep);
                }
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int v = lane + 32 * (i0 + i);
                float fa[8], fb[8];
                unpack8(wa[i], fa);
                unpack8(wb[i], fb);
#pragma unroll
                for (int b = 0; b < BM; b++) {
                    if (b < B) {
                        float xf[8];
                        unpack8(*reinterpret_cast<const uint4*>(xs + (size_t)b * K + v * 8), xf);
#pragma unroll
                        for (int j = 0; j < 8; j++) acc0[b] = fmaf(fa[j], xf[j], acc0[b]);
#pragma unroll
                        for (int j = 0; j < 8; j++) acc1[b] = fmaf(fb[j], xf[j], acc1[b]);
                    }
                }
            }
        }
        float my0 = 0.f, my1 = 0.f;      // lane b keeps the sums of batch row b
#pragma unroll
        for (int b = 0; b < BM; b++) {
            if (b < B) {
                const float s0 = warp_sum(acc0[b]), s1 = warp_sum(acc1[b]);
                if (lane == b) { my0 = s0; my1 = s1; }
            }
        }
        if (SWIGLU && lane < B) {
            const float g = bf16_round(my0), u = bf16_round(my1);
            y[(size_t)lane * ldy + r0] = __float2bfloat16_rn(bf16_round(silu_f(g)) * u);
        }
        if (!SWIGLU && lane < B) {
            const int b = lane;
            float o0 = my0, o1 = my1;
            if (res) {
                o0 = bf16_round(o0) + __bfloat162float(__ushort_as_bfloat16(res0));
                if (has1) o1 = bf16_round(o1) + __bfloat162float(__ushort_as_bfloat16(res1));
            }
            y[(size_t)b * ldy + r0] = __float2bfloat16_rn(o0);
            if (has1) y[(size_t)b * ldy + r1] = __float2bfloat16_rn(o1);
        }
    }
}

// ---- staging of the activations into shared memory (one warp per batch row) -------------------------------------
// Every loop below issues its global loads in batches of four 16-byte vectors per lane BEFORE using any of them (K = 1024 is
// exactly one batch): with a runtime trip count the compiler emits load -> use -> load -> use, i.e. one L2 round trip
// (300-600 cycles) per vector on the critical path of every phase.
// RMSNorm in place on a shared row (hf :62-67: fp32 statistics, round, times weight, round)
__device__ __forceinline__ void norm_row_inplace(bf16* row, int K, const bf16* __restrict__ w, float eps, int lane) {
    const int nvec = K / 8;
    float ss = 0.f;
    for (int v = lane; v < nvec; v += 32) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
        for (int j = 0; j < 8; j++) ss = fmaf(f[j], f[j], ss);
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)K + eps);
    for (int v0 = lane; v0 < nvec; v0 += 128) {
        uint4 wr[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
            if (v0 + 32 * i < nvec) wr[i] = *reinterpret_cast<const uint4*>(w + (v0 + 32 * i) * 8);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int v = v0 + 32 * i;
            if (v < nvec) {
                float f[8], wv[8];
                unpack8(*reinterpret_cast<const uint4*>(row + v * 8), f);
                unpack8(wr[i], wv);
#pragma unroll
                for (int j = 0; j < 8; j++) f[j] = wv[j] * bf16_round(f[j] * rstd);
                *reinterpret_cast<uint4*>(row + v * 8) = pack8(f);
            }
        }
    }
}
__device__ __forceinline__ void copy_row_from_global(bf16* dst, const bf16* src, int K, int lane) {
    const int nvec = K / 8;
    for (int v0 = lane; v0 < nvec; v0 += 128) {
        uint4 r[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
            if (v0 + 32 * i < nvec) r[i] = ldcg16(src + (v0 + 32 * i) * 8);
#pragma unroll
        for (int i = 0; i < 4; i++)
            if (v0 + 32 * i < nvec) *reinterpret_cast<uint4*>(dst + (v0 + 32 * i) * 8) = r[i];
    }
}
__device__ __forceinline__ void copy_row_to_global(bf16* dst, const bf16* src, int K, int lane) {
    for (int v = lane; v < K / 8; v += 32) *reinterpret_cast<uint4*>(dst + v * 8) = *reinterpret_cast<const uint4*>(src + v * 8);
}

// ---- event-level attention: one warp per (row, head, chunk of the context) ---------------------------------------
__device__ __forceinline__ size_t kv_base(const int* bt, int max_pages, int page, int nh, int D, int b, int h, int t) {
    const int pg = bt[b * max_pages + t / page];
    return (((size_t)pg * nh + h) * page + (t % page)) * D;
}

// The chunk grid of the batch-1 kernel over a context of T positions (outer_attention with B = 1): returns the chunk length
// and sets n_chunks.  The ROWS kernel cuts each row this way, so that the row's sums do not depend on the batch.
__device__ __forceinline__ int rows_grid(int T, int nh, int ngw, int& n_chunks) {
    const int target = min(PD_MAXC, max(1, ngw / nh));
    const int chunk = ((T + target - 1) / target + 31) / 32 * 32;
    n_chunks = (T + chunk - 1) / chunk;
    return chunk;
}

// RAGGED: row b's new position is pos + row_off[b] <= pos.  The chunk grid stays on the shared length pos + 1 (uniform
// across the grid), so the trailing chunks of a shorter row can be empty: their key loop does not run and they write the
// neutral partial (m = -inf, l = 0, o = 0), which the combine pass weights by exp(-inf - mx) = 0.  Chunk 0 is never empty.
// QUEUE: a row that is not live (row_last[b] != -1, written by CTA 0 at the last commit and read after a grid barrier)
// skips its items: it appends nothing and reads none of its pages.
// ROWS (implies QUEUE): each live row's context is cut as the batch-1 kernel cuts it at the row's own length (rows_grid),
// so its attention sums in the order of generating it alone; the items run over (b, h, c < n_chunks_b) of the live rows.
// A row with one chunk writes its output directly; n_chunks_out is the largest count of a live row, the same in every CTA.
template <bool RAGGED, bool QUEUE = false, bool ROWS = false>
__device__ __noinline__ void outer_attention(const PDArg<RAGGED, QUEUE, ROWS>& p, int layer, int pos_shared, int B, int gw,
                                                int ngw, int lane, float* q_s, bf16* kn_s, bf16* vn_s, int& n_chunks_out) {
    const DD& d = p.d;
    constexpr int D = 64;
    const int nh = d.nh_outer, H = d.H;
    const int T = pos_shared + 1;
    const int items = B * nh;
    int target = ngw / items;
    if (target < 1) target = 1;
    if (target > PD_MAXC) target = PD_MAXC;
    int chunk = (T + target - 1) / target;
    chunk = (chunk + 31) / 32 * 32;
    const int n_chunks = (T + chunk - 1) / chunk;
    n_chunks_out = n_chunks;
    int n_items = 0;                                     // ROWS: items of the live rows
    if constexpr (ROWS) {
        n_chunks_out = 1;
        for (int b = 0; b < B; b++) {
            if (__ldcg(p.row_last + b) != -1) continue;
            int nc;
            rows_grid(pos_shared + p.row_off[b] + 1, nh, ngw, nc);
            n_items += nh * nc;
            n_chunks_out = max(n_chunks_out, nc);
        }
    }
    bf16* kpool = reinterpret_cast<bf16*>(d.kv_outer[layer * 2 + 0]);
    bf16* vpool = reinterpret_cast<bf16*>(d.kv_outer[layer * 2 + 1]);
    const float scale = 0.125f;
    for (int it = gw; it < (ROWS ? n_items : items * n_chunks); it += ngw) {
        int bh = it / n_chunks, c = it % n_chunks;
        int b = bh / nh, h = bh % nh;
        int chunk_b = chunk, n_chunks_b = n_chunks;      // ROWS: the grid of row b
        if constexpr (ROWS) {
            int r = it;                                  // item r of the live rows' items, in row order
            for (b = 0;; b++) {
                if (__ldcg(p.row_last + b) != -1) continue;
                chunk_b = rows_grid(pos_shared + p.row_off[b] + 1, nh, ngw, n_chunks_b);
                if (r < nh * n_chunks_b) break;
                r -= nh * n_chunks_b;
            }
            h = r / n_chunks_b;
            c = r % n_chunks_b;
            bh = b * nh + h;
        } else if constexpr (QUEUE) {
            if (__ldcg(p.row_last + b) != -1) continue;
        }
        int pos = pos_shared;
        if constexpr (RAGGED) pos += p.row_off[b];
        const int t0 = c * chunk_b, t1 = min(pos + 1, t0 + chunk_b);
        const bf16* row = p.qkv + (size_t)b * 3 * H;
        const float cs = __bfloat162float(d.cos_outer[(size_t)pos * 32 + lane]), sn = __bfloat162float(d.sin_outer[(size_t)pos * 32 + lane]);
        {
            const float x1 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + h * D + lane))));
            const float x2 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + h * D + lane + 32))));
            q_s[lane] = bf16_round(rope_fwd_elem(x1, x2, cs, sn, false));
            q_s[lane + 32] = bf16_round(rope_fwd_elem(x2, x1, cs, sn, true));
        }
        const bool owns_new = (t0 <= pos && pos < t1);
        if (owns_new) {   // RoPE(k), v of the new position: used from shared memory here and appended to the cache
            const float x1 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + H + h * D + lane))));
            const float x2 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + H + h * D + lane + 32))));
            kn_s[lane] = __float2bfloat16_rn(rope_fwd_elem(x1, x2, cs, sn, false));
            kn_s[lane + 32] = __float2bfloat16_rn(rope_fwd_elem(x2, x1, cs, sn, true));
            vn_s[lane] = __ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + 2 * H + h * D + lane)));
            vn_s[lane + 32] = __ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + 2 * H + h * D + lane + 32)));
        }
        __syncwarp();
        if (owns_new) {
            const size_t o = kv_base(d.block_table, d.max_pages, d.page, nh, D, b, h, pos);
            if (lane < 8) *reinterpret_cast<uint4*>(kpool + o + lane * 8) = *reinterpret_cast<const uint4*>(kn_s + lane * 8);
            else if (lane < 16) *reinterpret_cast<uint4*>(vpool + o + (lane - 8) * 8) = *reinterpret_cast<const uint4*>(vn_s + (lane - 8) * 8);
        }
        // Scores: lane <-> key (the lane reads its key's 128-byte row).  P.V: 8 lanes per key, each with 8 of the 64 dims as one
        // 16-byte load -- key j = (lane >> 3) + 4 i, dims 8 (lane & 7) .. + 7 -- so a 32-key block is 8 + 8 vector loads per
        // lane, all issued together (one memory latency per block), then two shuffle steps fold the four key groups.
        const int kg = lane >> 3, dl = lane & 7;
        float m_run = -INFINITY, l_run = 0.f;
        float av[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int tb = t0; tb < t1; tb += 32) {
            const size_t base = kv_base(d.block_table, d.max_pages, d.page, nh, D, b, h, tb);   // 32-aligned: one page
            const int t = tb + lane;
            uint4 kr[8], vr[8];
#pragma unroll
            for (int dv = 0; dv < 8; dv++) {
                kr[dv] = make_uint4(0, 0, 0, 0);
                if (t < t1 && t != pos) kr[dv] = ldcg16(kpool + base + (size_t)lane * D + dv * 8);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int tj = tb + kg + 4 * i;
                vr[i] = make_uint4(0, 0, 0, 0);
                if (tj < t1 && tj != pos) vr[i] = ldcg16(vpool + base + (size_t)(kg + 4 * i) * D + dl * 8);
            }
            if (owns_new && pos >= tb && pos < tb + 32) {      // the new position's key / value come from shared memory
                if (t == pos) {
#pragma unroll
                    for (int dv = 0; dv < 8; dv++) kr[dv] = *reinterpret_cast<const uint4*>(kn_s + dv * 8);
                }
#pragma unroll
                for (int i = 0; i < 8; i++)
                    if (tb + kg + 4 * i == pos) vr[i] = *reinterpret_cast<const uint4*>(vn_s + dl * 8);
            }
            float s = -INFINITY;
            if (t < t1) {
                float acc = 0.f;
#pragma unroll
                for (int dv = 0; dv < 8; dv++) {
                    float kf[8];
                    unpack8(kr[dv], kf);
#pragma unroll
                    for (int j = 0; j < 8; j++) acc = fmaf(kf[j], q_s[dv * 8 + j], acc);
                }
                s = acc * scale;
            }
            const float m_new = fmaxf(m_run, warp_max(s));
            const float pr = (t < t1) ? __expf(s - m_new) : 0.f;
            const float corr = __expf(m_run - m_new);          // 0 on the first block (m_run = -inf)
            l_run = l_run * corr + warp_sum(pr);
            m_run = m_new;
            const float pb = bf16_round(pr);                    // P rounded to bf16 before P.V (flash semantics)
#pragma unroll
            for (int j = 0; j < 8; j++) av[j] *= corr;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float pj = __shfl_sync(0xffffffffu, pb, kg + 4 * i);     // 0 for keys past the chunk
                float vf[8];
                unpack8(vr[i], vf);
#pragma unroll
                for (int j = 0; j < 8; j++) av[j] = fmaf(pj, vf[j], av[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            av[j] += __shfl_xor_sync(0xffffffffu, av[j], 8);
            av[j] += __shfl_xor_sync(0xffffffffu, av[j], 16);
        }
        if (n_chunks_b == 1) {
            if (kg == 0) {
                const float inv = 1.f / l_run;
#pragma unroll
                for (int j = 0; j < 8; j++) av[j] *= inv;
                *reinterpret_cast<uint4*>(p.attn + (size_t)b * H + h * D + dl * 8) = pack8(av);
            }
        } else {
            float* po = p.partial + ((size_t)bh * PD_MAXC + c) * (D + 2);
            if (lane == 0) { po[0] = m_run; po[1] = l_run; }
            if (kg == 0) {
#pragma unroll
                for (int j = 0; j < 8; j++) po[2 + dl * 8 + j] = av[j];
            }
        }
        __syncwarp();
    }
}

__device__ __noinline__ void outer_attention_combine(const PD& p, int B, int n_chunks, int gw, int ngw, int lane) {
    constexpr int D = 64;
    const int nh = p.d.nh_outer, H = p.d.H;
    for (int bh = gw; bh < B * nh; bh += ngw) {
        const float* pp = p.partial + (size_t)bh * PD_MAXC * (D + 2);
        float mx = -INFINITY;
        for (int c = lane; c < n_chunks; c += 32) mx = fmaxf(mx, __ldcg(pp + c * (D + 2)));
        mx = warp_max(mx);
        float l = 0.f;
        for (int c = lane; c < n_chunks; c += 32) l += __ldcg(pp + c * (D + 2) + 1) * __expf(__ldcg(pp + c * (D + 2)) - mx);
        l = warp_sum(l);
        float a0 = 0.f, a1 = 0.f;
        for (int c = 0; c < n_chunks; c++) {
            const float w = __expf(__ldcg(pp + c * (D + 2)) - mx);
            const float2 o = __ldcg(reinterpret_cast<const float2*>(pp + c * (D + 2) + 2 + 2 * lane));
            a0 = fmaf(o.x, w, a0);
            a1 = fmaf(o.y, w, a1);
        }
        const int b = bh / nh, h = bh % nh;
        const float inv = 1.f / l;
        *reinterpret_cast<bf162*>(p.attn + (size_t)b * H + h * D + 2 * lane) = __floats2bfloat162_rn(a0 * inv, a1 * inv);
    }
}
// ROWS: each live row with more than one chunk combines exactly its own n_chunks_b partials (outer_attention)
__device__ __noinline__ void outer_attention_combine_rows(const PDRows& p, int pos_shared, int B, int gw, int ngw, int lane) {
    constexpr int D = 64;
    const int nh = p.d.nh_outer, H = p.d.H;
    for (int bh = gw; bh < B * nh; bh += ngw) {
        const int b = bh / nh;
        if (__ldcg(p.row_last + b) != -1) continue;
        int n_chunks;
        rows_grid(pos_shared + p.row_off[b] + 1, nh, ngw, n_chunks);
        if (n_chunks == 1) continue;
        // the arithmetic of outer_attention_combine for this (row, head), written out here so that the instructions of
        // that function (and of the kernels that call it) stay as they are
        const float* pp = p.partial + (size_t)bh * PD_MAXC * (D + 2);
        float mx = -INFINITY;
        for (int c = lane; c < n_chunks; c += 32) mx = fmaxf(mx, __ldcg(pp + c * (D + 2)));
        mx = warp_max(mx);
        float l = 0.f;
        for (int c = lane; c < n_chunks; c += 32) l += __ldcg(pp + c * (D + 2) + 1) * __expf(__ldcg(pp + c * (D + 2)) - mx);
        l = warp_sum(l);
        float a0 = 0.f, a1 = 0.f;
        for (int c = 0; c < n_chunks; c++) {
            const float w = __expf(__ldcg(pp + c * (D + 2)) - mx);
            const float2 o = __ldcg(reinterpret_cast<const float2*>(pp + c * (D + 2) + 2 + 2 * lane));
            a0 = fmaf(o.x, w, a0);
            a1 = fmaf(o.y, w, a1);
        }
        const int h = bh % nh;
        const float inv = 1.f / l;
        *reinterpret_cast<bf162*>(p.attn + (size_t)b * H + h * D + 2 * lane) = __floats2bfloat162_rn(a0 * inv, a1 * inv);
    }
}

// ---- token-level attention (context <= 8, head_dim 256): one warp per (row, head), as decode_attn_small_kernel -------
__device__ __noinline__ void inner_attention(const PD& p, int layer, int step, int B, int gw, int ngw, int lane) {
    const DD& d = p.d;
    constexpr int D = 256;
    const int nh = d.nh_inner, H = d.H;
    const float scale = 0.0625f;
    bf16* k2 = p.k2 + (size_t)layer * B * PD_T * H;
    bf16* v2 = p.v2 + (size_t)layer * B * PD_T * H;
    for (int wid = gw; wid < B * nh; wid += ngw) {
        const int b = wid / nh, h = wid % nh;
        const bf16* row = p.qkv + (size_t)b * 3 * H + h * D;
        float qv[8], kv_[8], cs[8], sn[8];
        unpack8(ldcg16(row + lane * 8), qv);
        unpack8(ldcg16(row + H + lane * 8), kv_);
        unpack8(*reinterpret_cast<const uint4*>(d.cos_inner + (size_t)step * (D / 2) + (lane & 15) * 8), cs);
        unpack8(*reinterpret_cast<const uint4*>(d.sin_inner + (size_t)step * (D / 2) + (lane & 15) * 8), sn);
        // q and k rotated in one loop, as in decode_attn_small_kernel: two calls of rope_fwd_lane spill 16 more bytes here
        float qr[8], kr[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float qo = __shfl_xor_sync(0xffffffffu, qv[j], 16), ko = __shfl_xor_sync(0xffffffffu, kv_[j], 16);
            qr[j] = bf16_round(rope_fwd_elem(qv[j], qo, cs[j], sn[j], lane >= 16));
            kr[j] = bf16_round(rope_fwd_elem(kv_[j], ko, cs[j], sn[j], lane >= 16));
        }
        const uint4 k_new = pack8(kr);
        const uint4 v_new = ldcg16(row + 2 * H + lane * 8);
        {
            const size_t o = ((size_t)b * PD_T + step) * H + h * D + lane * 8;
            *reinterpret_cast<uint4*>(k2 + o) = k_new;
            *reinterpret_cast<uint4*>(v2 + o) = v_new;
        }
        const int T = step + 1;
        // all cached keys / values of this head at once (<= 7 rows of 16 bytes per lane): one L2 latency, not T
        uint4 kraw[PD_T], vraw[PD_T];
#pragma unroll
        for (int t = 0; t < PD_T; t++) {
            if (t < step) {
                kraw[t] = ldcg16(k2 + ((size_t)b * PD_T + t) * H + h * D + lane * 8);
                vraw[t] = ldcg16(v2 + ((size_t)b * PD_T + t) * H + h * D + lane * 8);
            }
        }
        float my_s = -INFINITY;
#pragma unroll
        for (int t = 0; t < PD_T; t++) {
            if (t < T) {
                float kf[8];
                unpack8(t == step ? k_new : kraw[t], kf);
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < 8; j++) s = fmaf(kf[j], qr[j], s);
                s = warp_sum(s) * scale;
                if (lane == t) my_s = s;
            }
        }
        const float mx = warp_max(my_s);
        const float pr = (lane < T) ? __expf(my_s - mx) : 0.f;
        const float sum = warp_sum(pr);
        const float pb = bf16_round(pr);
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int t = 0; t < PD_T; t++) {
            if (t < T) {
                const float pt = __shfl_sync(0xffffffffu, pb, t);
                float vf[8];
                unpack8(t == step ? v_new : vraw[t], vf);
#pragma unroll
                for (int j = 0; j < 8; j++) acc[j] = fmaf(pt, vf[j], acc[j]);
            }
        }
        const float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] *= inv;
        *reinterpret_cast<uint4*>(p.attn + (size_t)b * H + h * D + lane * 8) = pack8(acc);
    }
}

// ---- sampling of one row by one CTA (sample_logits_kernel of decode.cu, for PD_THREADS threads) -------------------
// ROWS: row b's own temp / top_p / top_k instead of the descriptor's
template <bool ROWS = false>
__device__ __noinline__ int sample_row(const PD& p, int b, int step, long long ev0, float u, float* s_p, int* s_i, int* s_cnt, float* s_red) {
    const DD& d = p.d;
    const int V = d.V;
    int lo, hi;
    if (step == 0) {
        lo = d.eos_id; hi = d.eos_id + 1 + d.n_event_types;
    } else {
        const int e = (int)ev0 - (d.eos_id + 1);
        if (ev0 == d.eos_id || e < 0 || e >= d.n_event_types) { lo = d.pad_id; hi = d.pad_id + 1; }
        else {
            lo = d.lut[(e * 8 + (step - 1)) * 2];
            hi = d.lut[(e * 8 + (step - 1)) * 2 + 1];
            if (hi <= lo) { lo = d.pad_id; hi = d.pad_id + 1; }
        }
    }
    if constexpr (ROWS) {
        const PDRows& r = static_cast<const PDRows&>(p);
        return smp::sample_logits_row<PD_THREADS, true>(p.logits + (size_t)b * d.pitch, V, r.row_temp[b], r.row_top_p[b],
                                                        r.row_top_k[b], lo, hi, d.dense_mask ? d.dense_mask + (size_t)b * V : nullptr,
                                                        u, s_p, s_i, s_cnt, s_red, true);
    }
    return smp::sample_logits_row<PD_THREADS, true>(p.logits + (size_t)b * d.pitch, V, d.temp, d.top_p, d.top_k, lo, hi,
                                              d.dense_mask ? d.dense_mask + (size_t)b * V : nullptr, u, s_p, s_i, s_cnt, s_red,
                                              true);
}

__device__ __forceinline__ float rng_uniform(unsigned long long seed, unsigned long long c, int i) {
    return smp::counter_uniform(seed, c, (unsigned long long)i);
}

// Row group g of a launch whose per-row phases run in NG groups of at most BM rows: its first row b0 and its row count
// (<= 0: no such group).  With one group it is the whole batch.
template <int BM, int NG>
__device__ __forceinline__ int row_group(int g, int B, int& b0) {
    b0 = g * BM;
    return NG > 1 ? min(BM, B - b0) : B;
}

// =================================================================================================================
// QUEUE (implies RAGGED): each row stops on its own.  A live row finishes at the commit of an event that is EOS or lands on
// row_end[b]; a row that is not live commits nothing, takes no part in the token-step count and skips its attention items.
// ROWS (implies QUEUE): per-request rows.  Row b samples with its own settings and draws from its own key (PDRows), and its
// event-level attention is cut on its own length (outer_attention), so a row's events do not depend on the other rows.
// STREAM (implies ROWS): each committed event is also written to the host mirror out_events, followed by a system fence
// and a release store of committed[b], so the host reads it while the launch runs.  Once per event, after the last token
// step's sampling, thread 0 of CTA 0 reads the host's ctl with an acquire load and stores it in the workspace; every CTA
// reads that word after the commit barrier and, when it is nonzero, leaves after this event's commit through the same
// uniform exit as exit_on_done.  No CTA reads ctl itself: CTAs that saw different values would deadlock at the next
// grid barrier.  The kernel only samples ctl, it never waits on host memory.
// Batch: 1..16 rows; ROWS (and STREAM) take 1..32.  A ROWS launch of more than 16 rows runs with BM = 16 and every phase
// that holds rows in shared memory or registers (the staging and norm blocks, the projections with their residual and
// SwiGLU stores) runs twice, once per group of 16 rows, each time with the code of a 16-row launch: row b's arithmetic is
// that of the same row at any batch.  Each group re-reads the phase's weights (the token-level ones from L2).  Attention,
// the sampler CTAs (one per row) and the commit loop over all B rows directly.
template <int BM, bool RAGGED, bool QUEUE = false, bool ROWS = false, bool STREAM = false>
__global__ void __launch_bounds__(PD_THREADS, 1) decode_events_kernel(const PDArg<RAGGED, QUEUE, ROWS, STREAM> p) {
    static_assert(!QUEUE || RAGGED, "the queue kernel positions its rows through row_off");
    static_assert(!ROWS || QUEUE, "per-request rows are queue rows");
    static_assert(!STREAM || ROWS, "the streaming kernel is the per-request queue kernel");
    constexpr int NG = (ROWS && BM == 16) ? 2 : 1;                                 // row groups (row_group)
    extern __shared__ __align__(16) uint8_t pd_smem[];
    const DD& d = p.d;
    const int B = d.batch, H = d.H;
    bf16* xs = reinterpret_cast<bf16*>(pd_smem);                                    // [BM][k_max]
    float* s_p = reinterpret_cast<float*>(pd_smem + (size_t)BM * p.k_max * 2);      // sampler: probabilities
    int* s_i = reinterpret_cast<int*>(s_p + smp::SMP_MAXV);
    int* s_cnt = s_i + smp::SMP_MAXV;                                               // [PD_THREADS + 1]
    float* s_red = reinterpret_cast<float*>(s_cnt + PD_THREADS + 8);                // [64]
    float* q_all = s_red + 64;                                                      // [PD_WARPS][64]
    bf16* kn_all = reinterpret_cast<bf16*>(q_all + PD_WARPS * 64);                  // [PD_WARPS][64]
    bf16* vn_all = kn_all + PD_WARPS * 64;
    int* cur_ev = reinterpret_cast<int*>(vn_all + PD_WARPS * 64);                   // [B][8] event fed to the event-level stack
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ngw = gridDim.x * PD_WARPS;
    const int gw = warp * gridDim.x + blockIdx.x;      // interleave the CTAs: consecutive row pairs land on different SMs
    // projections run on warps 1..15: warp 0 owns the grid barrier and must not have weight prefetches in flight
    const int ngwv = gridDim.x * (PD_WARPS - 1);
    const int gwv = warp == 0 ? 0x3fffffff : (warp - 1) * gridDim.x + blockIdx.x;
    float* q_s = q_all + warp * 64;
    bf16* kn_s = kn_all + warp * 64;
    bf16* vn_s = vn_all + warp * 64;

    const unsigned long long pol_stream = l2_policy(false), pol_keep = l2_policy(true);
    GridBar gb{p.bar, 0u, gridDim.x};
    int pos = __ldcg(d.pos);
    for (int i = threadIdx.x; i < B * PD_T; i += PD_THREADS) cur_ev[i] = (int)__ldcg(d.ev_in + i);
    const unsigned long long rng_c0 = d.rng_state[0], rng_seed = d.rng_state[1];
    unsigned live = 0;                                  // QUEUE: bit b set while row b is live, the same in every thread
    if constexpr (QUEUE) {
        for (int b = 0; b < B; b++)
            if (__ldcg(p.row_last + b) == -1) live |= 1u << b;
    }
    __syncthreads();

    int events_done = 0;
    Pre pre;
    Prof prof{d.prof, clock64(), clock64()};
    for (int e = 0; e < p.n_events; e++) {
        if (pos + 1 >= d.max_len) break;
        // =============================== event-level stack: one new position per row ===============================
        for (int l = 0; l < d.n_outer; l++) {
            const LayerW w = layer_w(d.outer_w, l);
            // ---- norm + QKV
            prefetch_rows<false>(pre, w.qkv, H, 3 * H, gwv, lane, pol_stream);
            if (l > 0) { grid_sync(gb); prof.mark(PH_DOWN_O); }   // layer 0 reads only this CTA's copy of the event: no wait
            for (int g = 0; g < NG; g++) {
                int b0;
                const int Bg = row_group<BM, NG>(g, B, b0);
                if (NG > 1 && Bg <= 0) break;
                if (NG > 1 && g > 0) __syncthreads();        // the previous group's projection has read xs
                if (warp < Bg) {
                    const int rb = b0 + warp;
                    bf16* row = xs + (size_t)warp * H;
                    if (l == 0) {
                        // embed_tokens(x).sum(-2) (midi_model.py:145-146): fp32 accumulate over the 8 ids, one rounding
                        for (int v = lane; v < H / 8; v += 32) {
                            uint4 er[PD_T];
#pragma unroll
                            for (int t = 0; t < PD_T; t++) {      // the 8 embedding rows of the event: loads in flight together
                                const int id = cur_ev[rb * PD_T + t];
                                er[t] = make_uint4(0, 0, 0, 0);
                                if (id >= 0 && id < d.V) er[t] = *reinterpret_cast<const uint4*>(d.emb_outer + (size_t)id * H + v * 8);
                            }
                            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
                            for (int t = 0; t < PD_T; t++) {
                                float f[8];
                                unpack8(er[t], f);
#pragma unroll
                                for (int j = 0; j < 8; j++) acc[j] += f[j];
                            }
                            *reinterpret_cast<uint4*>(row + v * 8) = pack8(acc);
                        }
                        __syncwarp();
                        if (blockIdx.x == 0) copy_row_to_global(p.x + (size_t)rb * H, row, H, lane);
                    } else {
                        copy_row_from_global(row, p.x + (size_t)rb * H, H, lane);
                    }
                    __syncwarp();
                    norm_row_inplace(row, H, w.ln1, d.eps, lane);
                }
                __syncthreads();
                prof.sub(PH_QKV_O, 0);
                gemv_pairs<BM, false>(xs, H, w.qkv, H, 3 * H, Bg, nullptr, 0, p.qkv + (size_t)b0 * 3 * H, 3 * H, gwv, ngwv,
                                      lane, pre, pol_stream);
                prof.sub(PH_QKV_O, 1);
            }
            // ---- RoPE + KV append + attention over positions 0..pos
            grid_sync(gb);
            prof.mark(PH_QKV_O);
            int n_chunks;
            outer_attention<RAGGED, QUEUE, ROWS>(p, l, pos, B, gw, ngw, lane, q_s, kn_s, vn_s, n_chunks);
            prof.sub(PH_ATT_O, 1);
            if (n_chunks > 1) {
                grid_sync(gb);
                prof.mark(PH_ATT_O);
                if constexpr (ROWS) outer_attention_combine_rows(p, pos, B, gw, ngw, lane);
                else outer_attention_combine(p, B, n_chunks, gw, ngw, lane);
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_stream);
                grid_sync(gb);
                prof.mark(PH_CMB_O);
            } else {
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_stream);
                grid_sync(gb);
                prof.mark(PH_ATT_O);
            }
            // ---- o_proj + residual
            for (int g = 0; g < NG; g++) {
                int b0;
                const int Bg = row_group<BM, NG>(g, B, b0);
                if (NG > 1 && Bg <= 0) break;
                if (NG > 1 && g > 0) __syncthreads();
                if (warp < Bg) copy_row_from_global(xs + (size_t)warp * H, p.attn + (size_t)(b0 + warp) * H, H, lane);
                __syncthreads();
                prof.sub(PH_OPROJ_O, 0);
                gemv_pairs<BM, false>(xs, H, w.o, H, H, Bg, p.x + (size_t)b0 * H, H, p.h + (size_t)b0 * H, H, gwv, ngwv, lane,
                                      pre, pol_stream);
                prof.sub(PH_OPROJ_O, 1);
            }
            // ---- norm + gate|up + SwiGLU
            prefetch_rows<true>(pre, w.gu, H, d.I_outer, gwv, lane, pol_stream);
            grid_sync(gb);
            prof.mark(PH_OPROJ_O);
            for (int g = 0; g < NG; g++) {
                int b0;
                const int Bg = row_group<BM, NG>(g, B, b0);
                if (NG > 1 && Bg <= 0) break;
                if (NG > 1 && g > 0) __syncthreads();
                if (warp < Bg) {
                    copy_row_from_global(xs + (size_t)warp * H, p.h + (size_t)(b0 + warp) * H, H, lane);
                    __syncwarp();
                    norm_row_inplace(xs + (size_t)warp * H, H, w.ln2, d.eps, lane);
                }
                __syncthreads();
                prof.sub(PH_GU_O, 0);
                gemv_pairs<BM, true>(xs, H, w.gu, H, d.I_outer, Bg, nullptr, 0, p.act + (size_t)b0 * d.I_outer, d.I_outer, gwv,
                                     ngwv, lane, pre, pol_stream);
                prof.sub(PH_GU_O, 1);
            }
            // ---- down + residual
            prefetch_rows<false>(pre, w.down, d.I_outer, H, gwv, lane, pol_stream);
            grid_sync(gb);
            prof.mark(PH_GU_O);
            for (int g = 0; g < NG; g++) {
                int b0;
                const int Bg = row_group<BM, NG>(g, B, b0);
                if (NG > 1 && Bg <= 0) break;
                __syncthreads();
                if (warp < Bg)
                    copy_row_from_global(xs + (size_t)warp * d.I_outer, p.act + (size_t)(b0 + warp) * d.I_outer, d.I_outer, lane);
                __syncthreads();
                prof.sub(PH_DOWN_O, 0);
                gemv_pairs<BM, false>(xs, d.I_outer, w.down, d.I_outer, H, Bg, p.h + (size_t)b0 * H, H, p.x + (size_t)b0 * H, H,
                                      gwv, ngwv, lane, pre, pol_stream);
                prof.sub(PH_DOWN_O, 1);
            }
        }
        // =============================== token-level stack: up to 8 steps =========================================
        int n_steps = PD_T;
        for (int i = 0; i < PD_T; i++) {
            if (i >= n_steps) break;
            for (int l = 0; l < d.n_inner; l++) {
                const LayerW w = layer_w(d.inner_w, l);
                prefetch_rows<false>(pre, w.qkv, H, 3 * H, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(l > 0 ? PH_DOWN_I : (i > 0 ? PH_SAMPLE : PH_DOWN_O));
                if (i == 1 && l == 0) {
                    // how many token steps this event needs (midi_model.py:234-237: stop once every live row has all its
                    // parameters; two steps at least, like the reference's loop)
                    int need = 2;
                    for (int b = 0; b < B; b++) {
                        if constexpr (QUEUE) {
                            if (!((live >> b) & 1u)) continue;
                        }
                        const long long ev = __ldcg(p.ev_t + b);
                        const int et = (int)ev - (d.eos_id + 1);
                        if (ev == d.eos_id || et < 0 || et >= d.n_event_types) continue;
                        int np = 0;
                        for (int s = 0; s < PD_T - 1; s++)
                            if (d.lut[(et * 8 + s) * 2 + 1] > d.lut[(et * 8 + s) * 2]) np = s + 1;
                        need = max(need, np + 1);
                    }
                    n_steps = min(PD_T, need);
                }
                for (int g = 0; g < NG; g++) {
                    int b0;
                    const int Bg = row_group<BM, NG>(g, B, b0);
                    if (NG > 1 && Bg <= 0) break;
                    if (NG > 1 && g > 0) __syncthreads();
                    if (warp < Bg) {
                        const int rb = b0 + warp;
                        bf16* row = xs + (size_t)warp * H;
                        if (l == 0) {
                            if (i == 0) {          // hidden = final norm of the event-level stack (hf :421), midi_model.py:126
                                copy_row_from_global(row, p.x + (size_t)rb * H, H, lane);
                                __syncwarp();
                                norm_row_inplace(row, H, d.outer_norm, d.eps, lane);
                            } else {               // embedding of the token sampled at the previous step (midi_model.py:128)
                                long long id = __ldcg(p.ev_t + (size_t)(i - 1) * B + rb);
                                if (id < 0 || id >= d.V) id = 0;
                                copy_row_from_global(row, d.emb_inner + (size_t)id * H, H, lane);
                            }
                            __syncwarp();
                            if (blockIdx.x == 0) copy_row_to_global(p.x2 + (size_t)rb * H, row, H, lane);
                        } else {
                            copy_row_from_global(row, p.x2 + (size_t)rb * H, H, lane);
                        }
                        __syncwarp();
                        norm_row_inplace(row, H, w.ln1, d.eps, lane);
                    }
                    __syncthreads();
                    prof.sub(PH_QKV_I, 0);
                    gemv_pairs<BM, false>(xs, H, w.qkv, H, 3 * H, Bg, nullptr, 0, p.qkv + (size_t)b0 * 3 * H, 3 * H, gwv, ngwv,
                                          lane, pre, pol_keep);
                    prof.sub(PH_QKV_I, 1);
                }
                grid_sync(gb);
                prof.mark(PH_QKV_I);
                inner_attention(p, l, i, B, gw, ngw, lane);
                prof.sub(PH_ATT_I, 1);
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_ATT_I);
                for (int g = 0; g < NG; g++) {
                    int b0;
                    const int Bg = row_group<BM, NG>(g, B, b0);
                    if (NG > 1 && Bg <= 0) break;
                    if (NG > 1 && g > 0) __syncthreads();
                    if (warp < Bg) copy_row_from_global(xs + (size_t)warp * H, p.attn + (size_t)(b0 + warp) * H, H, lane);
                    __syncthreads();
                    prof.sub(PH_OPROJ_I, 0);
                    gemv_pairs<BM, false>(xs, H, w.o, H, H, Bg, p.x2 + (size_t)b0 * H, H, p.h2 + (size_t)b0 * H, H, gwv, ngwv,
                                          lane, pre, pol_keep);
                    prof.sub(PH_OPROJ_I, 1);
                }
                prefetch_rows<true>(pre, w.gu, H, d.I_inner, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_OPROJ_I);
                for (int g = 0; g < NG; g++) {
                    int b0;
                    const int Bg = row_group<BM, NG>(g, B, b0);
                    if (NG > 1 && Bg <= 0) break;
                    if (NG > 1 && g > 0) __syncthreads();
                    if (warp < Bg) {
                        copy_row_from_global(xs + (size_t)warp * H, p.h2 + (size_t)(b0 + warp) * H, H, lane);
                        __syncwarp();
                        norm_row_inplace(xs + (size_t)warp * H, H, w.ln2, d.eps, lane);
                    }
                    __syncthreads();
                    prof.sub(PH_GU_I, 0);
                    gemv_pairs<BM, true>(xs, H, w.gu, H, d.I_inner, Bg, nullptr, 0, p.act + (size_t)b0 * d.I_inner, d.I_inner,
                                         gwv, ngwv, lane, pre, pol_keep);
                    prof.sub(PH_GU_I, 1);
                }
                prefetch_rows<false>(pre, w.down, d.I_inner, H, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_GU_I);
                for (int g = 0; g < NG; g++) {
                    int b0;
                    const int Bg = row_group<BM, NG>(g, B, b0);
                    if (NG > 1 && Bg <= 0) break;
                    if (NG > 1 && g > 0) __syncthreads();
                    if (warp < Bg)
                        copy_row_from_global(xs + (size_t)warp * d.I_inner, p.act + (size_t)(b0 + warp) * d.I_inner, d.I_inner,
                                             lane);
                    __syncthreads();
                    prof.sub(PH_DOWN_I, 0);
                    gemv_pairs<BM, false>(xs, d.I_inner, w.down, d.I_inner, H, Bg, p.h2 + (size_t)b0 * H, H,
                                          p.x2 + (size_t)b0 * H, H, gwv, ngwv, lane, pre, pol_keep);
                    prof.sub(PH_DOWN_I, 1);
                }
            }
            // ---- final norm + lm_head
            prefetch_rows<false>(pre, d.lm_head, H, d.V, gwv, lane, pol_keep);
            grid_sync(gb);
            prof.mark(PH_DOWN_I);
            for (int g = 0; g < NG; g++) {
                int b0;
                const int Bg = row_group<BM, NG>(g, B, b0);
                if (NG > 1 && Bg <= 0) break;
                if (NG > 1 && g > 0) __syncthreads();
                if (warp < Bg) {
                    copy_row_from_global(xs + (size_t)warp * H, p.x2 + (size_t)(b0 + warp) * H, H, lane);
                    __syncwarp();
                    norm_row_inplace(xs + (size_t)warp * H, H, d.inner_norm, d.eps, lane);
                }
                __syncthreads();
                prof.sub(PH_LMHEAD, 0);
                gemv_pairs<BM, false>(xs, H, d.lm_head, H, d.V, Bg, nullptr, 0, p.logits + (size_t)b0 * d.pitch, d.pitch, gwv,
                                      ngwv, lane, pre, pol_keep);
                prof.sub(PH_LMHEAD, 1);
            }
            // ---- sample (one CTA per row): temperature softmax, grammar range, top-p / top-k, draw
            grid_sync(gb);
            prof.mark(PH_LMHEAD);
            if ((int)blockIdx.x < B) {
                const int b = blockIdx.x;
                bool sample = true;
                if constexpr (QUEUE) sample = (live >> b) & 1u;
                if (sample) {
                    const long long ev0 = (i == 0) ? 0 : __ldcg(p.ev_t + b);
                    float u;
                    if constexpr (ROWS) {       // the draw of generating the request alone: batch 1, row 0, its own seed
                        const int j = pos + p.row_off[b] - p.row_first[b];
                        u = rng_uniform(p.row_seed[b], (unsigned long long)(j * PD_T + i), 0);
                    } else {
                        u = rng_uniform(rng_seed, rng_c0 + (unsigned long long)(events_done * PD_T + i), b);
                    }
                    const int id = sample_row<ROWS>(p, b, i, ev0, u, s_p, s_i, s_cnt, s_red);
                    if (threadIdx.x == 0) p.ev_t[(size_t)i * B + b] = id;
                } else if (threadIdx.x == 0) {
                    p.ev_t[(size_t)i * B + b] = d.pad_id;     // a row that is not live draws nothing
                }
            }
            prof.sub(PH_SAMPLE, 1);
        }
        // =============================== commit the event ========================================================
        if constexpr (STREAM) {                          // published to every CTA by the barrier below
            if (blockIdx.x == 0 && threadIdx.x == 0) *p.ctl_seen = ld_acquire_sys_s32(p.ctl);
        }
        grid_sync(gb);                                   // every row's tokens are visible
        prof.mark(PH_SAMPLE);
        int leave = 0;                                   // STREAM: the same value in every thread of the grid
        if constexpr (STREAM) leave = __ldcg(p.ctl_seen);
        __syncthreads();
        for (int k = threadIdx.x; k < B * PD_T; k += PD_THREADS) {
            const int b = k / PD_T, t = k % PD_T;
            const long long v = (t < n_steps) ? __ldcg(p.ev_t + (size_t)t * B + b) : (long long)d.pad_id;
            cur_ev[k] = (int)v;
            bool commit = blockIdx.x == 0;
            if constexpr (QUEUE) commit = commit && ((live >> b) & 1u);
            if (commit) {
                int row_pos = pos;                        // RAGGED: row b commits at its own position
                if constexpr (RAGGED) row_pos += p.row_off[b];
                d.seq[((size_t)b * d.max_len + row_pos + 1) * PD_T + t] = v;
                d.ev_in[k] = v;
                if constexpr (STREAM) {
                    p.out_events[((size_t)b * d.max_len + row_pos + 1) * PD_T + t] = v;
                    __threadfence_system();
                }
            }
        }
        __syncthreads();
        if constexpr (STREAM) {                           // after every token of the row's event is fenced
            const int b = threadIdx.x;
            if (blockIdx.x == 0 && b < B && ((live >> b) & 1u)) st_release_sys_s32(p.committed + b, pos + p.row_off[b] + 1);
        }
        prof.mark(PH_COMMIT);
        unsigned fin = 0;                                 // QUEUE: rows that finished in this event
        if constexpr (QUEUE) {
            // Every thread of the grid derives the same finish flags from the same values (the event types, visible since
            // the barrier above, row_off and row_end), so the decision to leave is uniform without another barrier.
            for (int b = 0; b < B; b++) {
                if (!((live >> b) & 1u)) continue;
                const int last = pos + p.row_off[b] + 1;  // seq index of the event row b just committed
                if (cur_ev[b * PD_T] == d.eos_id || last >= p.row_end[b]) {
                    fin |= 1u << b;
                    if (blockIdx.x == 0 && threadIdx.x == 0) p.row_last[b] = last;
                }
            }
            live &= ~fin;
        }
        pos++;
        events_done++;
        if constexpr (QUEUE) {
            if (live == 0 || (fin != 0 && p.exit_on_done)) break;
        }
        if constexpr (STREAM) {
            if (leave) break;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *d.pos = pos;
        d.rng_state[0] = rng_c0 + (unsigned long long)events_done * PD_T;
    }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct WsLayout {
    size_t bar, x, h, x2, h2, qkv, attn, act, logits, ev_t, partial, k2, v2, total;
};
WsLayout ws_layout(const b200_decode_desc& d) {
    WsLayout L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    const size_t B = d.batch, H = d.H;
    const size_t imax = d.I_outer > d.I_inner ? d.I_outer : d.I_inner;
    L.bar = take(256);
    L.x = take(B * H * 2); L.h = take(B * H * 2); L.x2 = take(B * H * 2); L.h2 = take(B * H * 2);
    L.qkv = take(B * 3 * H * 2); L.attn = take(B * H * 2); L.act = take(B * imax * 2);
    L.logits = take(B * d.pitch * 2);
    L.ev_t = take(PD_T * B * 8);
    L.partial = take(B * d.nh_outer * (size_t)PD_MAXC * 66 * 4);
    L.k2 = take((size_t)d.n_inner * B * PD_T * H * 2);
    L.v2 = take((size_t)d.n_inner * B * PD_T * H * 2);
    L.total = o;
    return L;
}

}   // namespace

extern "C" size_t b200_decode_events_workspace_bytes(const b200_decode_desc* d) { return ws_layout(*d).total; }
extern "C" size_t b200_decode_desc_bytes(void) { return sizeof(b200_decode_desc); }

namespace {

// per-request settings of the ROWS kernel (b200_decode_events_queue_rows)
struct RowArgs {
    const float *temp, *top_p;
    const int* top_k;
    const unsigned long long* seed;
    const int* first;
};
// host mirror and control flag of the STREAM kernel (b200_decode_events_queue_stream), as device pointers
struct StreamArgs {
    long long* out_events;
    int* committed;
    const int* ctl;
};

template <bool RAGGED, bool QUEUE = false, bool ROWS = false, bool STREAM = false>
int decode_events(const b200_decode_desc* desc, const int* row_off, const int* row_end, int* row_last, int exit_on_done,
                  int n_events, void* workspace, size_t workspace_bytes, cudaStream_t stream, const RowArgs* rows = nullptr,
                  const StreamArgs* st = nullptr) {
    const b200_decode_desc& d = *desc;
    B200_CHECK_ARG(!RAGGED || row_off != nullptr, "decode_events_ragged: row_off required");
    B200_CHECK_ARG(!QUEUE || (row_end != nullptr && row_last != nullptr), "decode_events_queue: row_end and row_last required");
    B200_CHECK_ARG(!ROWS || (rows != nullptr && rows->temp != nullptr && rows->top_p != nullptr && rows->top_k != nullptr &&
                             rows->seed != nullptr && rows->first != nullptr),
                   "decode_events_queue_rows: row_temp, row_top_p, row_top_k, row_seed and row_first required");
    constexpr int max_batch = ROWS ? 32 : 16;           // per-request rows: two groups of 16 (decode_events_kernel)
    B200_CHECK_ARG(d.batch >= 1 && d.batch <= max_batch, "decode_events: batch %d outside 1..%d", d.batch, max_batch);
    B200_CHECK_ARG(d.H == 1024 && d.nh_outer * 64 == d.H && d.nh_inner * 256 == d.H,
                   "decode_events: built for hidden 1024 (16 x 64 event-level heads, 4 x 256 token-level heads)");
    B200_CHECK_ARG(d.I_outer % 256 == 0 && d.I_inner % 256 == 0, "decode_events: MLP widths must be multiples of 256");
    B200_CHECK_ARG(d.V <= smp::SMP_MAXV && d.pitch >= d.V, "decode_events: vocabulary %d unsupported", d.V);
    B200_CHECK_ARG(d.page % 32 == 0, "decode_events: KV page size must be a multiple of 32");
    B200_CHECK_ARG(d.temp > 0.f && d.top_k >= 1 && d.top_k <= smp::FAST_MAXK,
                   "decode_events: temperature must be positive and 1 <= top_k <= %d", smp::FAST_MAXK);
    if (n_events <= 0) return B200_OK;
    const WsLayout L = ws_layout(d);
    B200_CHECK_ARG(workspace != nullptr && workspace_bytes >= L.total && ((uintptr_t)workspace % 256 == 0),
                   "decode_events: workspace too small or misaligned (%zu < %zu)", workspace_bytes, L.total);
    uint8_t* ws = (uint8_t*)workspace;
    PD p;
    DD& t = p.d;
    t.outer_w = d.outer_w; t.inner_w = d.inner_w; t.n_outer = d.n_outer; t.n_inner = d.n_inner;
    t.outer_norm = (const bf16*)d.outer_norm; t.inner_norm = (const bf16*)d.inner_norm; t.lm_head = (const bf16*)d.lm_head;
    t.emb_outer = (const bf16*)d.emb_outer; t.emb_inner = (const bf16*)d.emb_inner;
    t.H = d.H; t.I_outer = d.I_outer; t.I_inner = d.I_inner; t.nh_outer = d.nh_outer; t.nh_inner = d.nh_inner;
    t.V = d.V; t.pitch = d.pitch; t.eps = d.eps;
    t.kv_outer = d.kv_outer; t.block_table = d.block_table; t.max_pages = d.max_pages; t.page = d.page;
    t.cos_outer = (const bf16*)d.cos_outer; t.sin_outer = (const bf16*)d.sin_outer;
    t.cos_inner = (const bf16*)d.cos_inner; t.sin_inner = (const bf16*)d.sin_inner;
    t.pos = d.pos; t.ev_in = d.ev_in; t.seq = d.seq; t.max_len = d.max_len; t.rng_state = d.rng_state;
    t.dense_mask = d.dense_mask; t.lut = d.lut; t.n_event_types = d.n_event_types; t.eos_id = d.eos_id; t.pad_id = d.pad_id;
    t.temp = d.temp; t.top_p = d.top_p; t.top_k = d.top_k; t.batch = d.batch;
    t.prof = d.prof;
    p.bar = (unsigned int*)(ws + L.bar);
    p.x = (bf16*)(ws + L.x); p.h = (bf16*)(ws + L.h); p.x2 = (bf16*)(ws + L.x2); p.h2 = (bf16*)(ws + L.h2);
    p.qkv = (bf16*)(ws + L.qkv); p.attn = (bf16*)(ws + L.attn); p.act = (bf16*)(ws + L.act);
    p.logits = (bf16*)(ws + L.logits);
    p.ev_t = (long long*)(ws + L.ev_t);
    p.partial = (float*)(ws + L.partial);
    p.k2 = (bf16*)(ws + L.k2); p.v2 = (bf16*)(ws + L.v2);
    p.n_events = n_events;
    p.k_max = d.I_outer > d.I_inner ? d.I_outer : d.I_inner;
    if (p.k_max < d.H) p.k_max = d.H;
    B200_CUDA(cudaMemsetAsync(p.bar, 0, 256, stream), "decode_events: barrier reset");
    PDArg<RAGGED, QUEUE, ROWS, STREAM> pk;
    static_cast<PD&>(pk) = p;
    if constexpr (RAGGED) pk.row_off = row_off;
    if constexpr (QUEUE) {
        pk.row_end = row_end;
        pk.row_last = row_last;
        pk.exit_on_done = exit_on_done;
    }
    if constexpr (ROWS) {
        pk.row_temp = rows->temp;
        pk.row_top_p = rows->top_p;
        pk.row_top_k = rows->top_k;
        pk.row_seed = rows->seed;
        pk.row_first = rows->first;
    }
    if constexpr (STREAM) {
        pk.out_events = st->out_events;
        pk.committed = st->committed;
        pk.ctl = st->ctl;
        pk.ctl_seen = (int*)(ws + L.bar + 128);      // in the barrier's 256 bytes, cleared with them before the launch
    }
    const int bm = d.batch <= 1 ? 1 : d.batch <= 2 ? 2 : d.batch <= 4 ? 4 : d.batch <= 8 ? 8 : 16;
    const size_t smem = (size_t)bm * p.k_max * 2 + (size_t)smp::SMP_MAXV * 8 + (PD_THREADS + 8) * 4 + 64 * 4 +
                        PD_WARPS * 64 * (4 + 2 + 2) + (size_t)(bm > d.batch ? bm : d.batch) * PD_T * 4 + 64;   // cur_ev: [B][8]
    void* args[] = {(void*)&pk};
    const void* fn = nullptr;
    switch (bm) {
        case 1: fn = (const void*)decode_events_kernel<1, RAGGED, QUEUE, ROWS, STREAM>; break;
        case 2: fn = (const void*)decode_events_kernel<2, RAGGED, QUEUE, ROWS, STREAM>; break;
        case 4: fn = (const void*)decode_events_kernel<4, RAGGED, QUEUE, ROWS, STREAM>; break;
        case 8: fn = (const void*)decode_events_kernel<8, RAGGED, QUEUE, ROWS, STREAM>; break;
        default: fn = (const void*)decode_events_kernel<16, RAGGED, QUEUE, ROWS, STREAM>; break;
    }
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "decode_events smem attr");
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, PD_THREADS, smem), "decode_events occupancy");
    B200_CHECK_ARG(per_sm >= 1, "decode_events: kernel does not fit on an SM (smem %zu)", smem);
    const int grid = b200_num_sms();       // one CTA per SM, all co-resident (cooperative launch)
    B200_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(PD_THREADS), args, smem, stream), "decode_events launch");
    b200_count_launches(1);
    return B200_OK;
}

}   // namespace

extern "C" int b200_decode_events(const b200_decode_desc* desc, int n_events, void* workspace, size_t workspace_bytes,
                                  cudaStream_t stream) {
    return decode_events<false>(desc, nullptr, nullptr, nullptr, 0, n_events, workspace, workspace_bytes, stream);
}

extern "C" int b200_decode_events_ragged(const b200_decode_desc* desc, const int* row_off, int n_events, void* workspace,
                                         size_t workspace_bytes, cudaStream_t stream) {
    return decode_events<true>(desc, row_off, nullptr, nullptr, 0, n_events, workspace, workspace_bytes, stream);
}

extern "C" int b200_decode_events_queue(const b200_decode_desc* desc, const int* row_off, const int* row_end, int* row_last,
                                        int exit_on_done, int n_events, void* workspace, size_t workspace_bytes,
                                        cudaStream_t stream) {
    return decode_events<true, true>(desc, row_off, row_end, row_last, exit_on_done, n_events, workspace, workspace_bytes,
                                     stream);
}

extern "C" int b200_decode_events_queue_rows(const b200_decode_desc* desc, const int* row_off, const int* row_end,
                                             int* row_last, int exit_on_done, int n_events, void* workspace,
                                             size_t workspace_bytes, const float* row_temp, const float* row_top_p,
                                             const int* row_top_k, const unsigned long long* row_seed, const int* row_first,
                                             cudaStream_t stream) {
    const RowArgs rows{row_temp, row_top_p, row_top_k, row_seed, row_first};
    return decode_events<true, true, true>(desc, row_off, row_end, row_last, exit_on_done, n_events, workspace,
                                           workspace_bytes, stream, &rows);
}

extern "C" int b200_decode_events_queue_stream(const b200_decode_desc* desc, const int* row_off, const int* row_end,
                                               int* row_last, int exit_on_done, int n_events, void* workspace,
                                               size_t workspace_bytes, const float* row_temp, const float* row_top_p,
                                               const int* row_top_k, const unsigned long long* row_seed,
                                               const int* row_first, long long* out_events, int* committed,
                                               const int* ctl, cudaStream_t stream) {
    B200_CHECK_ARG(out_events != nullptr && committed != nullptr && ctl != nullptr,
                   "decode_events_queue_stream: out_events, committed and ctl required (pinned host memory)");
    StreamArgs st{};
    void* dev = nullptr;
    B200_CUDA(cudaHostGetDevicePointer(&dev, (void*)out_events, 0), "decode_events_queue_stream: out_events is not pinned");
    st.out_events = (long long*)dev;
    B200_CUDA(cudaHostGetDevicePointer(&dev, (void*)committed, 0), "decode_events_queue_stream: committed is not pinned");
    st.committed = (int*)dev;
    B200_CUDA(cudaHostGetDevicePointer(&dev, (void*)ctl, 0), "decode_events_queue_stream: ctl is not pinned");
    st.ctl = (const int*)dev;
    const RowArgs rows{row_temp, row_top_p, row_top_k, row_seed, row_first};
    return decode_events<true, true, true, true>(desc, row_off, row_end, row_last, exit_on_done, n_events, workspace,
                                                 workspace_bytes, stream, &rows, &st);
}
