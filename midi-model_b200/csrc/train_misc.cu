// Loss and optimizer kernels of the train step:
//  * cross-entropy over the (event, token) double loss -- train.py:180-185: mean CE over all
//    M*8 token positions with ignore_index = pad (0); forward saves the row log-sum-exp, backward
//    overwrites the logits with d(loss)/d(logits) in place (no second 0.9 GB buffer).
//  * global grad-norm clip (train.py:464, gradient_clip_val=1.0) and AdamW with the no-decay
//    split (train.py:121-138) over ONE flat parameter / gradient buffer: one launch per step.
#include "common.cuh"

namespace {

constexpr int CE_THREADS = 128;

__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
    v = warp_max(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float t = sh[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); i++) t = fmaxf(t, sh[i]);
    return t;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += sh[i];
    return t;
}

// one CTA per row: lse[r] = logsumexp(logits[r, :V]); row_loss[r] = lse - logit[target] (0 if ignored)
__global__ void __launch_bounds__(CE_THREADS)
ce_fwd_kernel(const bf16* __restrict__ logits, const long long* __restrict__ targets, float* __restrict__ lse_out,
              float* __restrict__ row_loss, int V, int ld, long long ignore_index) {
    __shared__ float sh[8];
    const size_t r = blockIdx.x;
    const bf16* row = logits + r * ld;
    const int nvec = (V + 7) / 8;
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < nvec; v += CE_THREADS) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (v * 8 + j < V) mx = fmaxf(mx, f[j]);
    }
    mx = block_reduce_max(mx, sh);
    float sum = 0.f;
    for (int v = threadIdx.x; v < nvec; v += CE_THREADS) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (v * 8 + j < V) sum += __expf(f[j] - mx);
    }
    sum = block_reduce_sum(sum, sh);
    if (threadIdx.x == 0) {
        const float lse = mx + logf(sum);
        lse_out[r] = lse;
        const long long t = targets[r];
        row_loss[r] = (t == ignore_index || t < 0 || t >= V) ? 0.f : lse - __bfloat162float(row[t]);
    }
}

// Warp-per-row variant: the whole row (<= 16 vectors of 8 per lane, i.e. V <= 4096) is loaded ONCE into registers with all
// loads in flight, max and sum-of-exponentials are then two passes over registers, reductions are shuffles (no block
// barrier).  The CTA-per-row kernel above re-reads the row and goes through four __syncthreads per 6.8 KB row.
constexpr int CEW_WARPS = 4;
template <int VPL>
__global__ void __launch_bounds__(CEW_WARPS * 32, 8)
ce_fwd_warp_kernel(const bf16* __restrict__ logits, const long long* __restrict__ targets, float* __restrict__ lse_out,
                   float* __restrict__ row_loss, long long R, int V, int ld, long long ignore_index) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nvec = (V + 7) / 8;
    const int tail = V - (nvec - 1) * 8;              // valid elements of the last vector (1..8)
    constexpr int CH = 8;                             // vectors per lane in flight at a time (32 registers)
    for (long long r = (long long)blockIdx.x * CEW_WARPS + warp; r < R; r += (long long)gridDim.x * CEW_WARPS) {
        const bf16* row = logits + (size_t)r * ld;
        float m = -INFINITY, s = 0.f;                 // running max / sum of exp(x - m) of this lane (online softmax)
#pragma unroll
        for (int k0 = 0; k0 < VPL; k0 += CH) {
            uint4 raw[CH];
#pragma unroll
            for (int k = 0; k < CH; k++) {
                const int v = lane + 32 * (k0 + k);
                raw[k] = make_uint4(0xFF80FF80u, 0xFF80FF80u, 0xFF80FF80u, 0xFF80FF80u);   // -inf: contributes nothing
                if (k0 + k < VPL && v < nvec) raw[k] = ld_nc16(row + v * 8);
                if (v == nvec - 1 && tail < 8) {      // pad columns of the pitched row do not belong to the vocabulary
                    auto fix = [&](unsigned int w, int e0) -> unsigned int {
                        if (e0 >= tail) w = (w & 0xFFFF0000u) | 0xFF80u;
                        if (e0 + 1 >= tail) w = (w & 0x0000FFFFu) | 0xFF800000u;
                        return w;
                    };
                    raw[k].x = fix(raw[k].x, 0); raw[k].y = fix(raw[k].y, 2); raw[k].z = fix(raw[k].z, 4); raw[k].w = fix(raw[k].w, 6);
                }
            }
#pragma unroll
            for (int k = 0; k < CH; k++) {
                float f[8];
                unpack8(raw[k], f);
                float m8 = fmaxf(fmaxf(fmaxf(f[0], f[1]), fmaxf(f[2], f[3])), fmaxf(fmaxf(f[4], f[5]), fmaxf(f[6], f[7])));
                if (m8 > m) {                         // (never taken with m8 = -inf)
                    s *= __expf(m - m8);              // m = -inf: s is 0 and stays 0
                    m = m8;
                }
                if (m > -INFINITY) {
#pragma unroll
                    for (int j = 0; j < 8; j++) s += __expf(f[j] - m);
                }
            }
        }
        const float mx = warp_max(m);
        const float sum = warp_sum(m > -INFINITY ? s * __expf(m - mx) : 0.f);
        if (lane == 0) {
            const float lse = mx + logf(sum);
            lse_out[r] = lse;
            const long long t = targets[r];
            row_loss[r] = (t == ignore_index || t < 0 || t >= V) ? 0.f : lse - __bfloat162float(row[t]);
        }
    }
}

// single CTA: loss_sum = sum(row_loss), count = #(target != ignore); out[0] = mean loss, out[1] = count
__global__ void ce_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ targets, size_t R, int V,
                                 long long ignore_index, float* __restrict__ out) {
    __shared__ float sh[32];
    float s = 0.f, c = 0.f;
    for (size_t i = threadIdx.x; i < R; i += blockDim.x) {
        s += row_loss[i];
        const long long t = targets[i];
        c += (t == ignore_index || t < 0 || t >= V) ? 0.f : 1.f;
    }
    s = block_reduce_sum(s, sh);
    c = block_reduce_sum(c, sh);
    if (threadIdx.x == 0) {
        out[0] = c > 0.f ? s / c : 0.f;
        out[1] = c;
    }
}

// dlogits[r, c] = (softmax - onehot) * gscale / count   (0 for ignored rows and for pad columns V..ld_zero)
__global__ void __launch_bounds__(CE_THREADS)
ce_bwd_kernel(bf16* __restrict__ logits, const long long* __restrict__ targets, const float* __restrict__ lse_in,
              const float* __restrict__ loss_and_count, int V, int ld, int n_cols_store, long long ignore_index,
              float gscale, const void* __restrict__ gscale_dev, int gscale_is_bf16) {
    B200_PDL_TRIGGER();
    // upstream d(loss) as a device scalar (autograd hands it over as a tensor: no host sync to read it)
    if (gscale_dev) gscale *= gscale_is_bf16 ? __bfloat162float(*reinterpret_cast<const bf16*>(gscale_dev))
                                             : *reinterpret_cast<const float*>(gscale_dev);
    const size_t r = blockIdx.x;
    bf16* row = logits + r * ld;
    const long long t = targets[r];
    const bool live = !(t == ignore_index || t < 0 || t >= V);
    const float cnt = loss_and_count[1];
    const float sc = live ? gscale / fmaxf(cnt, 1.f) : 0.f;
    const float lse = lse_in[r];
    const int nvec = n_cols_store / 8;
    for (int v = threadIdx.x; v < nvec; v += CE_THREADS) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int c = v * 8 + j;
            float g = 0.f;
            if (live && c < V) g = (__expf(f[j] - lse) - (c == (int)t ? 1.f : 0.f)) * sc;
            f[j] = g;
        }
        *reinterpret_cast<uint4*>(row + v * 8) = pack8(f);
    }
}

// ---- grad norm / clip / AdamW over flat buffers ---------------------------------------------
__global__ void sumsq_kernel(const bf16* __restrict__ g, size_t n, float* __restrict__ partials) {
    __shared__ float sh[32];
    float s = 0.f;
    const size_t nv = n / 8;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
        float f[8];
        unpack8(ld_nc16(g + i * 8), f);
#pragma unroll
        for (int j = 0; j < 8; j++) s = fmaf(f[j], f[j], s);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0)
        for (size_t i = nv * 8; i < n; i++) { float x = __bfloat162float(g[i]); s = fmaf(x, x, s); }
    s = block_reduce_sum(s, sh);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}
// out[0] = ||g||_2, out[1] = clip coefficient min(1, max_norm / (norm + 1e-6))  (torch clip_grad_norm_)
__global__ void clip_coef_kernel(const float* __restrict__ partials, int n, float max_norm, float* __restrict__ out) {
    __shared__ float sh[32];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
    s = block_reduce_sum(s, sh);
    if (threadIdx.x == 0) {
        const float norm = sqrtf(s);
        out[0] = norm;
        float c = max_norm > 0.f ? max_norm / (norm + 1e-6f) : 1.f;
        out[1] = c < 1.f ? c : 1.f;
    }
}

// torch.optim.AdamW step (decoupled decay), fp32 moments, bf16 parameters and gradients.
// nodecay[i / 256] != 0 marks 256-element blocks that belong to a no-decay parameter.
__global__ void adamw_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             const unsigned char* __restrict__ nodecay, size_t n, float lr, float b1, float b2, float eps,
                             float wd, float bc1, float bc2_sqrt, const float* __restrict__ clip) {
    const float gs = clip ? clip[1] : 1.f;
    const size_t nv = n / 8;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
        float pf[8], gf[8];
        unpack8(*reinterpret_cast<const uint4*>(p + i * 8), pf);
        unpack8(ld_nc16(g + i * 8), gf);
        float4 m0 = *reinterpret_cast<const float4*>(m + i * 8), m1 = *reinterpret_cast<const float4*>(m + i * 8 + 4);
        float4 v0 = *reinterpret_cast<const float4*>(v + i * 8), v1 = *reinterpret_cast<const float4*>(v + i * 8 + 4);
        float mm[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
        float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        const float decay = nodecay[(i * 8) >> 8] ? 1.f : 1.f - lr * wd;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float gg = gf[j] * gs;
            mm[j] = b1 * mm[j] + (1.f - b1) * gg;
            vv[j] = b2 * vv[j] + (1.f - b2) * gg * gg;
            const float denom = sqrtf(vv[j]) / bc2_sqrt + eps;
            pf[j] = pf[j] * decay - (lr / bc1) * (mm[j] / denom);
        }
        *reinterpret_cast<uint4*>(p + i * 8) = pack8(pf);
        *reinterpret_cast<float4*>(m + i * 8) = make_float4(mm[0], mm[1], mm[2], mm[3]);
        *reinterpret_cast<float4*>(m + i * 8 + 4) = make_float4(mm[4], mm[5], mm[6], mm[7]);
        *reinterpret_cast<float4*>(v + i * 8) = make_float4(vv[0], vv[1], vv[2], vv[3]);
        *reinterpret_cast<float4*>(v + i * 8 + 4) = make_float4(vv[4], vv[5], vv[6], vv[7]);
    }
}

}   // namespace

extern "C" int b200_ce_fwd(const void* logits, const long long* targets, float* lse, float* row_loss, float* loss_and_count,
                           long long rows, int V, int ld, long long ignore_index, cudaStream_t stream) {
    B200_CHECK_ARG(ld % 8 == 0 && ld >= V, "ce_fwd: ld (%d) must be a multiple of 8 and >= V (%d)", ld, V);
    B200_CHECK_ARG(((V + 7) / 8) * 8 <= ld, "ce_fwd: row pitch too small for vector loads");
    if (rows > 0) {
        const int vpl = ((V + 7) / 8 + 31) / 32;          // 16-byte vectors per lane when one warp holds a row
        long long blocks = (rows + CEW_WARPS - 1) / CEW_WARPS;
        const long long cap = (long long)b200_num_sms() * 16;
        const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
#define B200_CE_FWDW(VPL) ce_fwd_warp_kernel<VPL><<<grid, CEW_WARPS * 32, 0, stream>>>((const bf16*)logits, targets, lse, row_loss, rows, V, ld, ignore_index)
        if (vpl <= 4) B200_CE_FWDW(4);
        else if (vpl <= 8) B200_CE_FWDW(8);
        else if (vpl <= 14) B200_CE_FWDW(14);
        else if (vpl <= 16) B200_CE_FWDW(16);
        else ce_fwd_kernel<<<(unsigned)rows, CE_THREADS, 0, stream>>>((const bf16*)logits, targets, lse, row_loss, V, ld, ignore_index);
#undef B200_CE_FWDW
        B200_CHECK_LAUNCH("ce_fwd");
    }
    ce_reduce_kernel<<<1, 1024, 0, stream>>>(row_loss, targets, (size_t)rows, V, ignore_index, loss_and_count);
    B200_CHECK_LAUNCH("ce_reduce");
    return B200_OK;
}

extern "C" int b200_ce_bwd(void* logits_inout, const long long* targets, const float* lse, const float* loss_and_count,
                           long long rows, int V, int ld, long long ignore_index, float grad_scale,
                           const void* grad_scale_dev, int grad_scale_is_bf16, cudaStream_t stream) {
    B200_CHECK_ARG(ld % 8 == 0 && ld >= V, "ce_bwd: ld must be a multiple of 8 and >= V");
    if (rows == 0) return B200_OK;
    const int n_cols_store = ((V + 7) / 8) * 8;
    ce_bwd_kernel<<<(unsigned)rows, CE_THREADS, 0, stream>>>((bf16*)logits_inout, targets, lse, loss_and_count, V, ld,
                                                             n_cols_store, ignore_index, grad_scale, grad_scale_dev,
                                                             grad_scale_is_bf16);
    B200_CHECK_LAUNCH("ce_bwd");
    return B200_OK;
}

extern "C" int b200_gradnorm_parts(void) { return b200_num_sms() * 8; }

// workspace: float[b200_gradnorm_parts()]; norm_and_coef: float[2] on device
extern "C" int b200_grad_clip_coef(const void* grads, long long n, float max_norm, float* norm_and_coef, void* workspace,
                                   size_t workspace_bytes, cudaStream_t stream) {
    const int parts = b200_gradnorm_parts();
    B200_CHECK_ARG(workspace_bytes >= parts * sizeof(float), "grad_clip_coef: workspace too small");
    B200_CHECK_ARG((uintptr_t)grads % 16 == 0, "grad_clip_coef: gradient buffer must be 16-byte aligned");
    sumsq_kernel<<<parts, 256, 0, stream>>>((const bf16*)grads, (size_t)n, (float*)workspace);
    B200_CHECK_LAUNCH("sumsq");
    clip_coef_kernel<<<1, 1024, 0, stream>>>((const float*)workspace, parts, max_norm, norm_and_coef);
    B200_CHECK_LAUNCH("clip_coef");
    return B200_OK;
}

extern "C" int b200_adamw_step(void* params, const void* grads, float* exp_avg, float* exp_avg_sq,
                               const unsigned char* nodecay_blocks, long long n, float lr, float beta1, float beta2,
                               float eps, float weight_decay, int step, const float* norm_and_coef, cudaStream_t stream) {
    B200_CHECK_ARG(n % 256 == 0, "adamw_step: flat buffer length must be a multiple of 256");
    B200_CHECK_ARG(step >= 1, "adamw_step: step counts from 1");
    if (n == 0) return B200_OK;
    const float bc1 = 1.f - powf(beta1, (float)step);
    const float bc2 = 1.f - powf(beta2, (float)step);
    const int grid = b200_num_sms() * 8;
    adamw_kernel<<<grid, 256, 0, stream>>>((bf16*)params, (const bf16*)grads, exp_avg, exp_avg_sq, nodecay_blocks,
                                           (size_t)n, lr, beta1, beta2, eps, weight_decay, bc1, sqrtf(bc2), norm_and_coef);
    B200_CHECK_LAUNCH("adamw_step");
    return B200_OK;
}
