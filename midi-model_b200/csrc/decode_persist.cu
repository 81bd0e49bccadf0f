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

#include "common.cuh"
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

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
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

__device__ __noinline__ void outer_attention(const PD& p, int layer, int pos, int B, int gw, int ngw, int lane,
                                                float* q_s, bf16* kn_s, bf16* vn_s, int& n_chunks_out) {
    const DD& d = p.d;
    constexpr int D = 64;
    const int nh = d.nh_outer, H = d.H;
    const int T = pos + 1;
    const int items = B * nh;
    int target = ngw / items;
    if (target < 1) target = 1;
    if (target > PD_MAXC) target = PD_MAXC;
    int chunk = (T + target - 1) / target;
    chunk = (chunk + 31) / 32 * 32;
    const int n_chunks = (T + chunk - 1) / chunk;
    n_chunks_out = n_chunks;
    bf16* kpool = reinterpret_cast<bf16*>(d.kv_outer[layer * 2 + 0]);
    bf16* vpool = reinterpret_cast<bf16*>(d.kv_outer[layer * 2 + 1]);
    const float scale = 0.125f;
    for (int it = gw; it < items * n_chunks; it += ngw) {
        const int bh = it / n_chunks, c = it % n_chunks;
        const int b = bh / nh, h = bh % nh;
        const int t0 = c * chunk, t1 = min(T, t0 + chunk);
        const bf16* row = p.qkv + (size_t)b * 3 * H;
        const float cs = __bfloat162float(d.cos_outer[(size_t)pos * 32 + lane]), sn = __bfloat162float(d.sin_outer[(size_t)pos * 32 + lane]);
        {
            const float x1 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + h * D + lane))));
            const float x2 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + h * D + lane + 32))));
            q_s[lane] = bf16_round(bf16_round(x1 * cs) + bf16_round(-x2 * sn));
            q_s[lane + 32] = bf16_round(bf16_round(x2 * cs) + bf16_round(x1 * sn));
        }
        const bool owns_new = (t0 <= pos && pos < t1);
        if (owns_new) {   // RoPE(k), v of the new position: used from shared memory here and appended to the cache
            const float x1 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + H + h * D + lane))));
            const float x2 = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(row + H + h * D + lane + 32))));
            kn_s[lane] = __float2bfloat16_rn(bf16_round(x1 * cs) + bf16_round(-x2 * sn));
            kn_s[lane + 32] = __float2bfloat16_rn(bf16_round(x2 * cs) + bf16_round(x1 * sn));
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
        if (n_chunks == 1) {
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
        const bool lo = lane < 16;
        float qr[8], kr[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float qo = __shfl_xor_sync(0xffffffffu, qv[j], 16), ko = __shfl_xor_sync(0xffffffffu, kv_[j], 16);
            qr[j] = bf16_round(bf16_round(qv[j] * cs[j]) + bf16_round((lo ? -qo : qo) * sn[j]));
            kr[j] = bf16_round(bf16_round(kv_[j] * cs[j]) + bf16_round((lo ? -ko : ko) * sn[j]));
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
    return smp::sample_logits_row<PD_THREADS, true>(p.logits + (size_t)b * d.pitch, V, d.temp, d.top_p, d.top_k, lo, hi,
                                              d.dense_mask ? d.dense_mask + (size_t)b * V : nullptr, u, s_p, s_i, s_cnt, s_red,
                                              true);
}

__device__ __forceinline__ float rng_uniform(unsigned long long seed, unsigned long long c, int i) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ULL * (c * 4096ULL + (unsigned long long)i + 1ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// =================================================================================================================
template <int BM>
__global__ void __launch_bounds__(PD_THREADS, 1) decode_events_kernel(const PD p) {
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
    int* cur_ev = reinterpret_cast<int*>(vn_all + PD_WARPS * 64);                   // [BM][8] event fed to the event-level stack
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
            if (warp < B) {
                bf16* row = xs + (size_t)warp * H;
                if (l == 0) {
                    // embed_tokens(x).sum(-2) (midi_model.py:145-146): fp32 accumulate over the 8 ids, one rounding
                    for (int v = lane; v < H / 8; v += 32) {
                        uint4 er[PD_T];
#pragma unroll
                        for (int t = 0; t < PD_T; t++) {      // the 8 embedding rows of the event: loads in flight together
                            const int id = cur_ev[warp * PD_T + t];
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
                    if (blockIdx.x == 0) copy_row_to_global(p.x + (size_t)warp * H, row, H, lane);
                } else {
                    copy_row_from_global(row, p.x + (size_t)warp * H, H, lane);
                }
                __syncwarp();
                norm_row_inplace(row, H, w.ln1, d.eps, lane);
            }
            __syncthreads();
            prof.sub(PH_QKV_O, 0);
            gemv_pairs<BM, false>(xs, H, w.qkv, H, 3 * H, B, nullptr, 0, p.qkv, 3 * H, gwv, ngwv, lane, pre, pol_stream);
            prof.sub(PH_QKV_O, 1);
            // ---- RoPE + KV append + attention over positions 0..pos
            grid_sync(gb);
            prof.mark(PH_QKV_O);
            int n_chunks;
            outer_attention(p, l, pos, B, gw, ngw, lane, q_s, kn_s, vn_s, n_chunks);
            prof.sub(PH_ATT_O, 1);
            if (n_chunks > 1) {
                grid_sync(gb);
                prof.mark(PH_ATT_O);
                outer_attention_combine(p, B, n_chunks, gw, ngw, lane);
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_stream);
                grid_sync(gb);
                prof.mark(PH_CMB_O);
            } else {
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_stream);
                grid_sync(gb);
                prof.mark(PH_ATT_O);
            }
            // ---- o_proj + residual
            if (warp < B) copy_row_from_global(xs + (size_t)warp * H, p.attn + (size_t)warp * H, H, lane);
            __syncthreads();
            prof.sub(PH_OPROJ_O, 0);
            gemv_pairs<BM, false>(xs, H, w.o, H, H, B, p.x, H, p.h, H, gwv, ngwv, lane, pre, pol_stream);
            prof.sub(PH_OPROJ_O, 1);
            // ---- norm + gate|up + SwiGLU
            prefetch_rows<true>(pre, w.gu, H, d.I_outer, gwv, lane, pol_stream);
            grid_sync(gb);
            prof.mark(PH_OPROJ_O);
            if (warp < B) {
                copy_row_from_global(xs + (size_t)warp * H, p.h + (size_t)warp * H, H, lane);
                __syncwarp();
                norm_row_inplace(xs + (size_t)warp * H, H, w.ln2, d.eps, lane);
            }
            __syncthreads();
            prof.sub(PH_GU_O, 0);
            gemv_pairs<BM, true>(xs, H, w.gu, H, d.I_outer, B, nullptr, 0, p.act, d.I_outer, gwv, ngwv, lane, pre, pol_stream);
            prof.sub(PH_GU_O, 1);
            // ---- down + residual
            prefetch_rows<false>(pre, w.down, d.I_outer, H, gwv, lane, pol_stream);
            grid_sync(gb);
            prof.mark(PH_GU_O);
            __syncthreads();
            if (warp < B) copy_row_from_global(xs + (size_t)warp * d.I_outer, p.act + (size_t)warp * d.I_outer, d.I_outer, lane);
            __syncthreads();
            prof.sub(PH_DOWN_O, 0);
            gemv_pairs<BM, false>(xs, d.I_outer, w.down, d.I_outer, H, B, p.h, H, p.x, H, gwv, ngwv, lane, pre, pol_stream);
            prof.sub(PH_DOWN_O, 1);
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
                if (warp < B) {
                    bf16* row = xs + (size_t)warp * H;
                    if (l == 0) {
                        if (i == 0) {          // hidden = final norm of the event-level stack (hf :421), midi_model.py:126
                            copy_row_from_global(row, p.x + (size_t)warp * H, H, lane);
                            __syncwarp();
                            norm_row_inplace(row, H, d.outer_norm, d.eps, lane);
                        } else {               // embedding of the token sampled at the previous step (midi_model.py:128)
                            long long id = __ldcg(p.ev_t + (size_t)(i - 1) * B + warp);
                            if (id < 0 || id >= d.V) id = 0;
                            copy_row_from_global(row, d.emb_inner + (size_t)id * H, H, lane);
                        }
                        __syncwarp();
                        if (blockIdx.x == 0) copy_row_to_global(p.x2 + (size_t)warp * H, row, H, lane);
                    } else {
                        copy_row_from_global(row, p.x2 + (size_t)warp * H, H, lane);
                    }
                    __syncwarp();
                    norm_row_inplace(row, H, w.ln1, d.eps, lane);
                }
                __syncthreads();
                prof.sub(PH_QKV_I, 0);
                gemv_pairs<BM, false>(xs, H, w.qkv, H, 3 * H, B, nullptr, 0, p.qkv, 3 * H, gwv, ngwv, lane, pre, pol_keep);
                prof.sub(PH_QKV_I, 1);
                grid_sync(gb);
                prof.mark(PH_QKV_I);
                inner_attention(p, l, i, B, gw, ngw, lane);
                prof.sub(PH_ATT_I, 1);
                prefetch_rows<false>(pre, w.o, H, H, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_ATT_I);
                if (warp < B) copy_row_from_global(xs + (size_t)warp * H, p.attn + (size_t)warp * H, H, lane);
                __syncthreads();
                prof.sub(PH_OPROJ_I, 0);
                gemv_pairs<BM, false>(xs, H, w.o, H, H, B, p.x2, H, p.h2, H, gwv, ngwv, lane, pre, pol_keep);
                prof.sub(PH_OPROJ_I, 1);
                prefetch_rows<true>(pre, w.gu, H, d.I_inner, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_OPROJ_I);
                if (warp < B) {
                    copy_row_from_global(xs + (size_t)warp * H, p.h2 + (size_t)warp * H, H, lane);
                    __syncwarp();
                    norm_row_inplace(xs + (size_t)warp * H, H, w.ln2, d.eps, lane);
                }
                __syncthreads();
                prof.sub(PH_GU_I, 0);
                gemv_pairs<BM, true>(xs, H, w.gu, H, d.I_inner, B, nullptr, 0, p.act, d.I_inner, gwv, ngwv, lane, pre, pol_keep);
                prof.sub(PH_GU_I, 1);
                prefetch_rows<false>(pre, w.down, d.I_inner, H, gwv, lane, pol_keep);
                grid_sync(gb);
                prof.mark(PH_GU_I);
                if (warp < B) copy_row_from_global(xs + (size_t)warp * d.I_inner, p.act + (size_t)warp * d.I_inner, d.I_inner, lane);
                __syncthreads();
                prof.sub(PH_DOWN_I, 0);
                gemv_pairs<BM, false>(xs, d.I_inner, w.down, d.I_inner, H, B, p.h2, H, p.x2, H, gwv, ngwv, lane, pre, pol_keep);
                prof.sub(PH_DOWN_I, 1);
            }
            // ---- final norm + lm_head
            prefetch_rows<false>(pre, d.lm_head, H, d.V, gwv, lane, pol_keep);
            grid_sync(gb);
            prof.mark(PH_DOWN_I);
            if (warp < B) {
                copy_row_from_global(xs + (size_t)warp * H, p.x2 + (size_t)warp * H, H, lane);
                __syncwarp();
                norm_row_inplace(xs + (size_t)warp * H, H, d.inner_norm, d.eps, lane);
            }
            __syncthreads();
            prof.sub(PH_LMHEAD, 0);
            gemv_pairs<BM, false>(xs, H, d.lm_head, H, d.V, B, nullptr, 0, p.logits, d.pitch, gwv, ngwv, lane, pre, pol_keep);
            prof.sub(PH_LMHEAD, 1);
            // ---- sample (one CTA per row): temperature softmax, grammar range, top-p / top-k, draw
            grid_sync(gb);
            prof.mark(PH_LMHEAD);
            if ((int)blockIdx.x < B) {
                const int b = blockIdx.x;
                const long long ev0 = (i == 0) ? 0 : __ldcg(p.ev_t + b);
                const float u = rng_uniform(rng_seed, rng_c0 + (unsigned long long)(events_done * PD_T + i), b);
                const int id = sample_row(p, b, i, ev0, u, s_p, s_i, s_cnt, s_red);
                if (threadIdx.x == 0) p.ev_t[(size_t)i * B + b] = id;
            }
            prof.sub(PH_SAMPLE, 1);
        }
        // =============================== commit the event ========================================================
        grid_sync(gb);                                   // every row's tokens are visible
        prof.mark(PH_SAMPLE);
        __syncthreads();
        for (int k = threadIdx.x; k < B * PD_T; k += PD_THREADS) {
            const int b = k / PD_T, t = k % PD_T;
            const long long v = (t < n_steps) ? __ldcg(p.ev_t + (size_t)t * B + b) : (long long)d.pad_id;
            cur_ev[k] = (int)v;
            if (blockIdx.x == 0) {
                d.seq[((size_t)b * d.max_len + pos + 1) * PD_T + t] = v;
                d.ev_in[k] = v;
            }
        }
        __syncthreads();
        prof.mark(PH_COMMIT);
        pos++;
        events_done++;
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

extern "C" int b200_decode_events(const b200_decode_desc* desc, int n_events, void* workspace, size_t workspace_bytes,
                                  cudaStream_t stream) {
    const b200_decode_desc& d = *desc;
    B200_CHECK_ARG(d.batch >= 1 && d.batch <= 16, "decode_events: batch %d outside 1..16", d.batch);
    B200_CHECK_ARG(d.H == 1024 && d.nh_outer * 64 == d.H && d.nh_inner * 256 == d.H,
                   "decode_events: built for hidden 1024 (16 x 64 event-level heads, 4 x 256 token-level heads)");
    B200_CHECK_ARG(d.I_outer % 256 == 0 && d.I_inner % 256 == 0, "decode_events: MLP widths must be multiples of 256");
    B200_CHECK_ARG(d.V <= smp::SMP_MAXV && d.pitch >= d.V, "decode_events: vocabulary %d unsupported", d.V);
    B200_CHECK_ARG(d.page % 32 == 0, "decode_events: KV page size must be a multiple of 32");
    B200_CHECK_ARG(d.temp > 0.f && d.top_k >= 1 && d.top_k <= 64, "decode_events: temperature must be positive and 1 <= top_k <= 64");
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
    const int bm = d.batch <= 1 ? 1 : d.batch <= 2 ? 2 : d.batch <= 4 ? 4 : d.batch <= 8 ? 8 : 16;
    const size_t smem = (size_t)bm * p.k_max * 2 + (size_t)smp::SMP_MAXV * 8 + (PD_THREADS + 8) * 4 + 64 * 4 +
                        PD_WARPS * 64 * (4 + 2 + 2) + (size_t)bm * PD_T * 4 + 64;
    void* args[] = {(void*)&p};
    const void* fn = nullptr;
    switch (bm) {
        case 1: fn = (const void*)decode_events_kernel<1>; break;
        case 2: fn = (const void*)decode_events_kernel<2>; break;
        case 4: fn = (const void*)decode_events_kernel<4>; break;
        case 8: fn = (const void*)decode_events_kernel<8>; break;
        default: fn = (const void*)decode_events_kernel<16>; break;
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
