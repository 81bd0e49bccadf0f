// Sampling helpers shared by the generate-loop kernels (decode.cu: one launch per token; decode_persist.cu: inside the
// persistent per-event kernel): compaction of the non-zero probabilities, histogram top-k preselection, bitonic sort,
// top-p on the un-renormalised mass + top-k + draw (midi_model.py:152-165).  NT = threads of the calling CTA.
#pragma once
#include "common.cuh"

namespace smp {

constexpr int SMP_MAXV = 4096;

// ---------------------------------------------------------------------------------------------
// sampler
// ---------------------------------------------------------------------------------------------

// The generate loops' counter-based uniform in [0, 1): draw i of counter value c under `seed` (a splitmix64 finaliser).
__device__ __forceinline__ float counter_uniform(unsigned long long seed, unsigned long long c, unsigned long long i) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ULL * (c * 4096ULL + i + 1ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}

__device__ __forceinline__ bool key_before(float pa, int ia, float pb, int ib) {   // sort order: prob desc, id asc
    return (pa > pb) || (pa == pb && ia < ib);
}

// Shared tail: s_p/s_i hold `n` candidate (prob, id) pairs (prob > 0), unsorted.  Sort, apply top-p on the
// un-renormalised mass and top-k, renormalise, draw with uniform u.  Returns the chosen id (all threads).
template <int NT>
__device__ int sample_tail(float* s_p, int* s_i, int n, float top_p, int top_k, float u, bool bf16_sem) {
    int n_sort = 32;
    while (n_sort < n) n_sort <<= 1;
    for (int i = n + threadIdx.x; i < n_sort; i += blockDim.x) { s_p[i] = -1.f; s_i[i] = 0x7fffffff; }
    __syncthreads();
    for (int k = 2; k <= n_sort; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_sort; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const bool up = (i & k) == 0;
                    const float pa = s_p[i], pb = s_p[ixj];
                    const int ia = s_i[i], ib = s_i[ixj];
                    const bool a_first = key_before(pa, ia, pb, ib);
                    if (up ? !a_first : a_first) { s_p[i] = pb; s_p[ixj] = pa; s_i[i] = ib; s_i[ixj] = ia; }
                }
            }
            __syncthreads();
        }
    }
    // Only ranks < kk can survive.  Sequential scan by one thread over <= kk entries is cheap for the
    // usual top_k (20); large k falls back to the same loop (still correct).
    const int kk = min(n, top_k);
    __shared__ int s_choice;
    if (threadIdx.x == 0) {
        float cum = 0.f, total = 0.f;
        const float pth = bf16_sem ? bf16_round(top_p) : top_p;
        int last = 0;
        for (int i = 0; i < kk; i++) {
            const float pi = s_p[i];
            cum += pi;
            const float cs = bf16_sem ? bf16_round(cum) : cum;
            const float before = bf16_sem ? bf16_round(cs - pi) : cs - pi;
            const float w = (before > pth) ? 0.f : pi;   // midi_model.py:155-156
            s_p[i] = w;   // weights overwrite the sorted probabilities in place
            total += w;
            if (w > 0.f) last = i;
        }
        int choice = 0;
        if (total > 0.f) {
            const float target = u * total;
            float run = 0.f;
            choice = last;
            for (int i = 0; i <= last; i++) {
                run += s_p[i];
                if (s_p[i] > 0.f && run > target) { choice = i; break; }
            }
        }
        s_choice = (n > 0) ? s_i[choice] : 0;
    }
    __syncthreads();
    return s_choice;
}

// compact the non-zero entries of s_p (indexed by id) into the front of (s_p, s_i); returns count.
template <int NT>
__device__ int compact_nonzero(float* s_p, int* s_i, int V, int* s_cnt) {
    const int per = (V + NT - 1) / NT;
    const int beg = threadIdx.x * per;
    const int end = min(V, beg + per);
    float loc_p[SMP_MAXV / NT];
    int c = 0;
    for (int i = beg; i < end; i++) {
        const float p = s_p[i];
        loc_p[i - beg] = p;
        if (p > 0.f) c++;
    }
    s_cnt[threadIdx.x] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int i = 0; i < NT; i++) { const int t = s_cnt[i]; s_cnt[i] = run; run += t; }
        s_cnt[NT] = run;
    }
    __syncthreads();
    int pos = s_cnt[threadIdx.x];
    const int total = s_cnt[NT];
    __syncthreads();   // everyone has read its chunk of s_p into registers before it is overwritten
    for (int i = beg; i < end; i++) {
        const float p = loc_p[i - beg];
        if (p > 0.f) { s_p[pos] = p; s_i[pos] = i; pos++; }
    }
    __syncthreads();
    return total;
}


// Top-k preselection: the sampling tail only looks at ranks < top_k, so instead of sorting all n candidates we keep the
// ones at or above the k-th largest value (found with two shared-memory histograms over the fp32 bit pattern: exponent,
// then the 8 mantissa bits below it -- probabilities are bf16-rounded so 8 mantissa bits separate all distinct values)
// and sort only those.  Returns the new candidate count (n itself when the selection would not shrink the set).
template <int NT>
__device__ int preselect_topk(float* s_p, int* s_i, int n, int top_k, int* s_hist /*[257]*/) {
    if (n <= 64 || top_k >= n || top_k > 64) return n;
    __shared__ int s_sel[2];       // {exponent bin, mantissa bin} of the k-th largest value
    __shared__ int s_count;
    for (int i = threadIdx.x; i < 257; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&s_hist[(__float_as_uint(s_p[i]) >> 23) & 0xFF], 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int cum = 0, e = 255;
        for (; e > 0; e--) { cum += s_hist[e]; if (cum >= top_k) break; }
        s_sel[0] = e;
        s_hist[256] = cum - s_hist[e];      // candidates strictly above the boundary exponent
    }
    __syncthreads();
    const int e_star = s_sel[0];
    const int above = s_hist[256];
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned u = __float_as_uint(s_p[i]);
        if (((u >> 23) & 0xFF) == (unsigned)e_star) atomicAdd(&s_hist[(u >> 15) & 0xFF], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int cum = above, m = 255;
        for (; m > 0; m--) { cum += s_hist[m]; if (cum >= top_k) break; }
        s_sel[1] = m;
        s_count = 0;
    }
    __syncthreads();
    const unsigned thr = ((unsigned)e_star << 23) | ((unsigned)s_sel[1] << 15);     // keep p with bit pattern >= thr
    // count first: if the selection is not small, keep everything
    int mine = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) mine += (__float_as_uint(s_p[i]) >= thr) ? 1 : 0;
    atomicAdd(&s_count, mine);
    __syncthreads();
    const int m_sel = s_count;
    __syncthreads();
    if (m_sel > 256 || m_sel >= n) return n;
    // compact the selected entries to the front (their order is fixed later by the (prob desc, id asc) sort)
    float keep_p[SMP_MAXV / NT];
    int keep_i[SMP_MAXV / NT];
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (__float_as_uint(s_p[i]) >= thr) { keep_p[c] = s_p[i]; keep_i[c] = s_i[i]; c++; }
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    const int base = atomicAdd(&s_count, c);
    __syncthreads();       // all reads of s_p / s_i are done (values are in registers) before the overwrite
    for (int j = 0; j < c; j++) { s_p[base + j] = keep_p[j]; s_i[base + j] = keep_i[j]; }
    __syncthreads();
    return m_sel;
}


// ---------------------------------------------------------------------------------------------
// Whole-row sampler: logits row -> token id, all NT threads of the CTA.
//   x = bf16(l / temp); p = bf16(exp(x - max) / sum) over the FULL vocabulary (midi_model.py:222: the mask is applied to
//   the softmax output, so the denominator covers every id); ids outside [lo, hi) or masked out get p = 0;
//   candidates sorted by (p desc, id asc); only the first min(n, top_k) can be drawn (midi_model.py:157-159); top-p on the
//   un-renormalised cumulative mass (:153-156); renormalise; draw with the uniform u (:161-164).
// Fast path (top_k <= 128, the default is 20): the top-k set is found with a 4-pass radix select over the 16-bit bf16
// patterns of p (per-warp shared-memory histograms), ties at the k-th value are resolved towards the lowest ids with a
// block-wide exclusive scan in id order, the <= 128 survivors are rank-sorted, one thread walks them.  ~17 block barriers
// instead of the ~60 (and three serial single-thread scans) of compaction + two histogram passes + a full bitonic sort.
// Results are identical to the general path (sample_tail on the compacted candidates), which remains for top_k > 128.
// Scratch: s_p [SMP_MAXV] floats, s_i [SMP_MAXV] ints, s_cnt [NT + 8] ints, s_red [64] floats; NT >= FAST_MAXK.
// ---------------------------------------------------------------------------------------------
constexpr int FAST_MAXK = 128;                          // largest top_k of the fast path

template <int NT, bool FAST_ONLY = false>
__device__ int sample_logits_row(const bf16* __restrict__ logits, int V, float temp, float top_p, int top_k, int lo, int hi,
                                 const unsigned char* __restrict__ mrow, float u, float* s_p, int* s_i, int* s_cnt,
                                 float* s_red, bool coherent_loads) {
    constexpr int NW = NT / 32;
    constexpr int PER = SMP_MAXV / NT;                 // ids per thread (consecutive: thread t owns [t * PER, t * PER + PER))
    static_assert(NT >= FAST_MAXK && 4 * NW * 16 + 4 * FAST_MAXK <= SMP_MAXV, "fast path: rank sort or survivors do not fit");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float mx = -INFINITY;
    {
        // the row's logits (<= PER per thread) requested together, then scaled / stored: one memory latency, not PER
        unsigned short lraw[PER];
#pragma unroll
        for (int k = 0; k < PER; k++) {
            const int i = tid + k * NT;
            lraw[k] = 0;
            if (i < V) lraw[k] = coherent_loads ? __ldcg(reinterpret_cast<const unsigned short*>(logits + i))
                                                : *reinterpret_cast<const unsigned short*>(logits + i);
        }
        const float inv_t = 1.f / temp;
        const bool unit = temp == 1.f;
#pragma unroll
        for (int k = 0; k < PER; k++) {
            const int i = tid + k * NT;
            if (i < V) {
                const float l = __bfloat162float(__ushort_as_bfloat16(lraw[k]));
                const float x = unit ? l : bf16_round(l / temp);
                s_p[i] = x;
                mx = fmaxf(mx, x);
            }
        }
        (void)inv_t;
    }
    mx = warp_max(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < NW; w++) mx = fmaxf(mx, s_red[w]);
    float sum = 0.f;
    for (int i = tid; i < V; i += NT) sum += __expf(s_p[i] - mx);
    sum = warp_sum(sum);
    if (lane == 0) s_red[32 + warp] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int w = 0; w < NW; w++) sum += s_red[32 + w];
    const float inv = 1.f / sum;

    if (!FAST_ONLY && top_k > FAST_MAXK) {             // general path
        __syncthreads();
        for (int i = tid; i < V; i += NT) {
            bool ok = (i >= lo && i < hi);
            if (ok && mrow) ok = mrow[i] != 0;
            s_p[i] = ok ? bf16_round(__expf(s_p[i] - mx) * inv) : 0.f;
        }
        __syncthreads();
        int n = compact_nonzero<NT>(s_p, s_i, V, s_cnt);
        if (n == 0) return lo;
        n = preselect_topk<NT>(s_p, s_i, n, top_k, s_cnt);
        return sample_tail<NT>(s_p, s_i, n, top_p, top_k, u, true);
    }

    // ---- fast path.  key = bf16 bit pattern of p (monotonic in p for p > 0), 0 = not a candidate
    unsigned key[PER];
    const int id0 = tid * PER;
    unsigned char mk[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {                     // mask bytes of this thread's ids, requested together
        const int id = id0 + j;
        mk[j] = 1;
        if (mrow != nullptr && id >= lo && id < hi && id < V) mk[j] = mrow[id];
    }
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const int id = id0 + j;
        unsigned k = 0;
        if (id >= lo && id < hi && id < V && mk[j] != 0) {
            const float pr = bf16_round(__expf(s_p[id] - mx) * inv);
            k = __float_as_uint(pr) >> 16;
        }
        key[j] = k;
    }
    int* hist = s_i;                                    // [4 passes][NW][16] per-warp digit histograms
    int* ctl = s_cnt;                                   // [0] prefix, [1] remaining, [2] n_pos; warp scan totals from [8]
    for (int i = tid; i < 4 * NW * 16; i += NT) hist[i] = 0;
    if (tid == 0) { ctl[0] = 0; ctl[1] = 0; ctl[2] = 0; }
    __syncthreads();
    unsigned prefix = 0;
    int remaining = 0, kk = 0;
#pragma unroll
    for (int pass = 0; pass < 4; pass++) {
        const int shift = 12 - 4 * pass;
        int* h = hist + (pass * NW + warp) * 16;
#pragma unroll
        for (int j = 0; j < PER; j++) {
            const unsigned k = key[j];
            if (k != 0 && (pass == 0 || (k >> (shift + 4)) == (prefix >> (shift + 4)))) atomicAdd(&h[(k >> shift) & 15], 1);
        }
        __syncthreads();
        if (warp == 0) {
            int c = 0;
            if (lane < 16)
                for (int w = 0; w < NW; w++) c += hist[(pass * NW + w) * 16 + lane];
            // suffix sums over the 16 bins: above(b) = candidates whose digit is > b
            int incl = c;
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) {
                const int t = __shfl_down_sync(0xffffffffu, incl, o);
                if (lane + o < 16) incl += t;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 0);
            int rem = remaining;
            if (pass == 0) {
                kk = min(total, top_k);
                rem = kk;
            }
            const int above = incl - c;
            const bool mine = lane < 16 && c > 0 && above < rem && rem <= incl;
            const unsigned ball = __ballot_sync(0xffffffffu, mine);
            if (pass == 0 && lane == 0) ctl[2] = total;
            if (ball != 0 && lane == (int)(__ffs(ball) - 1)) {
                ctl[0] = (int)(prefix | ((unsigned)lane << shift));
                ctl[1] = rem - above;
            }
        }
        __syncthreads();
        prefix = (unsigned)ctl[0];
        remaining = ctl[1];
        if (pass == 0) {
            if (ctl[2] == 0) return lo;                 // every allowed probability underflowed (reference: multinomial raises)
            kk = min(ctl[2], top_k);
        }
    }
    const unsigned thr = prefix;                        // key of the kk-th largest candidate
    const int need_ties = remaining;                    // how many of the candidates equal to thr are inside the top kk
    // ---- exclusive scan in id order of (#keys > thr, #keys == thr)
    int c_gt = 0, c_eq = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) {
        c_gt += key[j] > thr ? 1 : 0;
        c_eq += (key[j] == thr && thr != 0) ? 1 : 0;
    }
    int packed = c_gt | (c_eq << 16);
    int incl = packed;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) ctl[8 + warp] = incl;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; w++) base += ctl[8 + w];
    const int excl = base + incl - packed;
    int gt_before = excl & 0xFFFF, eq_before = excl >> 16;
    // survivors in s_i past the digit histograms (read for the last time before the scan's barrier)
    float* sel_p = reinterpret_cast<float*>(hist + 4 * NW * 16);          // [FAST_MAXK]
    int* sel_i = hist + 4 * NW * 16 + FAST_MAXK;                          // [FAST_MAXK]
    float* srt_p = reinterpret_cast<float*>(hist + 4 * NW * 16 + 2 * FAST_MAXK);   // [FAST_MAXK]
    int* srt_i = hist + 4 * NW * 16 + 3 * FAST_MAXK;                      // [FAST_MAXK]
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const unsigned k = key[j];
        if (k > thr) {
            const int pos = gt_before + min(eq_before, need_ties);
            sel_p[pos] = __uint_as_float(k << 16);
            sel_i[pos] = id0 + j;
            gt_before++;
        } else if (k == thr && thr != 0) {
            if (eq_before < need_ties) {
                const int pos = gt_before + eq_before;
                sel_p[pos] = __uint_as_float(k << 16);
                sel_i[pos] = id0 + j;
            }
            eq_before++;
        }
    }
    __syncthreads();
    // ---- rank sort of the kk survivors by (p desc, id asc)
    if (tid < kk) {
        const float pm = sel_p[tid];
        const int im = sel_i[tid];
        int rank = 0;
        for (int j = 0; j < kk; j++) rank += key_before(sel_p[j], sel_i[j], pm, im) ? 1 : 0;
        srt_p[rank] = pm;
        srt_i[rank] = im;
    }
    __syncthreads();
    if (tid == 0) {
        float cum = 0.f, total = 0.f;
        const float pth = bf16_round(top_p);
        int last = 0;
        for (int i = 0; i < kk; i++) {
            const float pi = srt_p[i];
            cum += pi;
            const float cs = bf16_round(cum);
            const float before = bf16_round(cs - pi);
            const float w = (before > pth) ? 0.f : pi;   // midi_model.py:155-156
            srt_p[i] = w;
            total += w;
            if (w > 0.f) last = i;
        }
        int choice = 0;
        if (total > 0.f) {
            const float target = u * total;
            float run = 0.f;
            choice = last;
            for (int i = 0; i <= last; i++) {
                run += srt_p[i];
                if (srt_p[i] > 0.f && run > target) { choice = i; break; }
            }
        }
        ctl[3] = srt_i[choice];
    }
    __syncthreads();
    return ctl[3];
}

}   // namespace smp
