// The six training losses of the reference (models/base.py:90-249, called from
// models/nersemble_instant_ngp.py:366-407) and their gradients w.r.t. the render outputs, fused.
//
// All six are functions of per-ray outputs (rgb, accumulation, depth) and of per-ray scans of the sample weights.
// The reference evaluates them with ~25 torch launches forward and as many in autograd, boolean-index gathers with host
// synchronisation, float64 cumulative sums over all samples and the torch_efficient_distloss extension.  Here:
//   losses_fwd_kernel   warp per ray: one pass over the ray's samples with shuffle scans; partial sums and counts
//                       go to 16 double accumulators (atomicAdd, 13 per ray) -> losses_finalize_kernel -> 6 values
//   losses_bwd_kernel   warp per ray: d rgb / d acc / d depth per ray and d weights per sample (prefix AND suffix sums of
//                       the ray: a reverse pass for the suffixes between two forward passes), scaled by the upstream
//                       gradient of each loss value
// Formulas (S = samples, R = rays; masks are 0/1; every mean divides by max(count, 1) except the rgb loss, which keeps
// the reference's 0/0 = nan for an empty mask):
//   rgb    mean over masked rays and 3 channels of (image - rgb)^2                 mask = alpha > alpha_mask_threshold
//   alpha  lambda_a * mean_{alpha < 1} |acc - alpha|
//   empty  lambda_e * mean_{tgt > 0, mid < tgt - eps} w^2                                          (training)
//   near   lambda_n * mean_{tgt > 0, |mid - tgt| <= eps} (A - Phi(mid - tgt))^2,  A = inclusive scan of w along the ray,
//          Phi = CDF of Normal(0, scale = (eps / 3)^2)   [sic: the reference passes the variance as scale]   (training)
//   depth  lambda_d * mean_{tgt > 0} (tgt - depth)^2                                                (training)
//   dist   lambda_dist / n_sel * sum_{rays < dist_max_rays} [ 1/3 sum d w^2 + 2 sum w (m W_pre - WM_pre) ]
//          (torch_efficient_distloss.flatten_eff_distloss; n_sel = largest selected ray index + 1)
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ float lw_incl_scan(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
// exclusive scans: the sum over the lanes below (prefix) or above (suffix) this one
__device__ __forceinline__ float lw_excl_scan(float v, int lane) {
    float x = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 0) x = 0.f;
    return lw_incl_scan(x, lane);
}
__device__ __forceinline__ float lw_excl_suffix(float v, int lane) {
    float x = __shfl_down_sync(0xffffffffu, v, 1);
    if (lane == 31) x = 0.f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_down_sync(0xffffffffu, x, o);
        if (lane + o < 32) x += t;
    }
    return x;
}
__device__ __forceinline__ float lw_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

enum { A_RGB = 0, A_NMASK, A_ALPHA, A_NBG, A_EMPTY, A_NVN, A_NEAR, A_NNEAR, A_DEPTH, A_NDM, A_D1, A_D2, A_MAXSEL, A_COUNT = 16 };

struct LossK {
    nsb_loss_args a;
};

__device__ __forceinline__ float normal_cdf(float x, float scale) { return 0.5f * (1.0f + erff(x / (scale * 1.4142135623730951f))); }

__global__ void __launch_bounds__(256) losses_fwd_kernel(const __grid_constant__ LossK K) {
    const nsb_loss_args &a = K.a;
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
    const bool depth_terms = a.depth_target != nullptr;
    const float tgt = depth_terms ? a.depth_target[ray] : 0.f;
    const bool sel = ray < a.dist_max_rays;
    const float scale = (a.eps_depth / 3.0f) * (a.eps_depth / 3.0f);
    float s_empty = 0.f, n_vn = 0.f, s_near = 0.f, n_near = 0.f, d1 = 0.f, d2 = 0.f;
    float cw = 0.f, cwm = 0.f;   // running inclusive sums of w and w*m over the previous chunks
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
        const float w = ok ? a.weights[s] : 0.f;
        const float m = (ts + te) * 0.5f;
        const float iw = lw_incl_scan(w, lane), iwm = lw_incl_scan(w * m, lane);
        const float A = cw + iw;                                  // inclusive
        const float Wpre = A - w, WMpre = cwm + iwm - w * m;      // exclusive
        if (ok) {
            if (depth_terms && tgt > 0.f) {
                if (a.lambda_empty > 0.f && m < tgt - a.eps_depth) { s_empty += w * w; n_vn += 1.f; }
                if (a.lambda_near > 0.f && tgt - a.eps_depth <= m && m <= tgt + a.eps_depth) {
                    const float r = A - normal_cdf(m - tgt, scale);
                    s_near += r * r; n_near += 1.f;
                }
            }
            if (sel) { d1 += (te - ts) * w * w; d2 += w * (m * Wpre - WMpre); }
        }
        cw += __shfl_sync(0xffffffffu, iw, 31);
        cwm += __shfl_sync(0xffffffffu, iwm, 31);
    }
    s_empty = lw_sum(s_empty); n_vn = lw_sum(n_vn); s_near = lw_sum(s_near); n_near = lw_sum(n_near);
    d1 = lw_sum(d1); d2 = lw_sum(d2);
    if (lane == 0) {
        double *acc = a.accum;
        if (n_vn > 0.f) { atomicAdd(acc + A_EMPTY, (double)s_empty); atomicAdd(acc + A_NVN, (double)n_vn); }
        if (n_near > 0.f) { atomicAdd(acc + A_NEAR, (double)s_near); atomicAdd(acc + A_NNEAR, (double)n_near); }
        if (sel && cnt > 0) {
            atomicAdd(acc + A_D1, (double)d1); atomicAdd(acc + A_D2, (double)d2);
            atomicMax(reinterpret_cast<unsigned long long *>(acc + A_MAXSEL), (unsigned long long)ray);
        }
        // per-ray terms
        const float al = a.alpha ? a.alpha[ray] : 1.0f;
        const bool masked = !(a.use_masked_rgb && a.alpha) || al > a.alpha_mask_threshold;
        if (masked) {
            float e = 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) { const float d = a.image[3 * ray + c] - a.rgb[3 * ray + c]; e += d * d; }
            atomicAdd(acc + A_RGB, (double)e); atomicAdd(acc + A_NMASK, 1.0);
        }
        if (a.lambda_alpha > 0.f && a.alpha && al < 1.0f) { atomicAdd(acc + A_ALPHA, (double)fabsf(a.acc[ray] - al)); atomicAdd(acc + A_NBG, 1.0); }
        if (a.lambda_depth > 0.f && depth_terms && tgt > 0.f) {
            const float d = tgt - a.depth[ray];
            atomicAdd(acc + A_DEPTH, (double)(d * d)); atomicAdd(acc + A_NDM, 1.0);
        }
    }
}

// values[6] = rgb, alpha, empty, near, depth, dist;  coef[8] = the per-element factors the backward multiplies with
__global__ void losses_finalize_kernel(const __grid_constant__ LossK K) {
    const nsb_loss_args &a = K.a;
    if (threadIdx.x != 0) return;
    const double *acc = a.accum;
    auto cnt1 = [](double n) { return n > 1.0 ? n : 1.0; };
    float *v = a.values, *c = a.coef;
    v[0] = (float)(acc[A_RGB] / (3.0 * acc[A_NMASK]));                       // 0/0 = nan for an empty mask (like torch's mean)
    v[1] = (float)(a.lambda_alpha * acc[A_ALPHA] / cnt1(acc[A_NBG]));
    v[2] = (float)(a.lambda_empty * acc[A_EMPTY] / cnt1(acc[A_NVN]));
    v[3] = (float)(a.lambda_near * acc[A_NEAR] / cnt1(acc[A_NNEAR]));
    v[4] = (float)(a.lambda_depth * acc[A_DEPTH] / cnt1(acc[A_NDM]));
    const double n_sel = (double)(*reinterpret_cast<const unsigned long long *>(acc + A_MAXSEL)) + 1.0;
    v[5] = (float)(a.lambda_dist * ((1.0 / 3.0) * acc[A_D1] + 2.0 * acc[A_D2]) / n_sel);
    c[0] = (float)(-2.0 / (3.0 * acc[A_NMASK]));           // d rgb_loss / d rgb = c0 * (image - rgb) on masked rays
    c[1] = (float)(a.lambda_alpha / cnt1(acc[A_NBG]));     // * sign(acc - alpha)
    c[2] = (float)(2.0 * a.lambda_empty / cnt1(acc[A_NVN]));   // * w
    c[3] = (float)(2.0 * a.lambda_near / cnt1(acc[A_NNEAR]));  // * suffix sum of (A - Phi) over near samples
    c[4] = (float)(-2.0 * a.lambda_depth / cnt1(acc[A_NDM]));  // * (tgt - depth)
    c[5] = (float)(a.lambda_dist / n_sel);
}

__global__ void __launch_bounds__(256) losses_bwd_kernel(const __grid_constant__ LossK K) {
    const nsb_loss_args &a = K.a;
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    const float *g = a.upstream, *c = a.coef;      // upstream gradient of each of the six values
    const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
    const bool depth_terms = a.depth_target != nullptr;
    const float tgt = depth_terms ? a.depth_target[ray] : 0.f;
    const bool sel = ray < a.dist_max_rays;
    const float scale = (a.eps_depth / 3.0f) * (a.eps_depth / 3.0f);
    if (lane == 0) {
        const float al = a.alpha ? a.alpha[ray] : 1.0f;
        const bool masked = !(a.use_masked_rgb && a.alpha) || al > a.alpha_mask_threshold;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
            a.d_rgb[3 * ray + ch] = masked ? g[0] * c[0] * (a.image[3 * ray + ch] - a.rgb[3 * ray + ch]) : 0.f;
        float da = 0.f;
        if (a.lambda_alpha > 0.f && a.alpha && al < 1.0f) {
            const float d = a.acc[ray] - al;
            da = g[1] * c[1] * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        }
        a.d_acc[ray] = da;
        a.d_depth[ray] = (a.lambda_depth > 0.f && depth_terms && tgt > 0.f) ? g[4] * c[4] * (tgt - a.depth[ray]) : 0.f;
    }
    if (cnt == 0) return;
    const float ce = g[2] * c[2], cn = g[3] * c[3], cd = g[5] * c[5];
    const bool want_near = depth_terms && tgt > 0.f && a.lambda_near > 0.f, want_empty = depth_terms && tgt > 0.f && a.lambda_empty > 0.f;
    // Every sum over earlier or later samples is its own scan (exclusive prefix front to back, suffix back to front), never
    // a difference of a total and a prefix: where the true sum is 0 (e.g. no near sample behind k) it then is exactly 0.
    // The samples' partial gradients are parked in their own d_weights slots between the passes (same thread).
    // pass 1, front to back (near loss only): the near residuals r_i = (A_i - Phi_i) * near_i, A = inclusive scan of w
    if (want_near) {
        float cw = 0.f;
        for (int64_t b = 0; b < cnt; b += 32) {
            const int64_t i = b + lane;
            const bool ok = i < cnt;
            const int64_t s = start + (ok ? i : 0);
            const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
            const float w = ok ? a.weights[s] : 0.f;
            const float m = (ts + te) * 0.5f;
            const float A = cw + lw_incl_scan(w, lane);
            cw = __shfl_sync(0xffffffffu, A, 31);
            if (ok) a.d_weights[s] = (tgt - a.eps_depth <= m && m <= tgt + a.eps_depth) ? A - normal_cdf(m - tgt, scale) : 0.f;
        }
    }
    // pass 2, back to front: near  cn * sum_{i >= k} r_i   (A_i depends on w_k for all i >= k)
    //                        dist  cd * 2 * sum_{i > k} w_i (m_i - m_k)
    if (want_near || sel) {
        float cr = 0.f, cw = 0.f, cwm = 0.f;   // suffix sums of the later chunks
        for (int64_t b = ((cnt - 1) >> 5) << 5; b >= 0; b -= 32) {
            const int64_t i = b + lane;
            const bool ok = i < cnt;
            const int64_t s = start + (ok ? i : 0);
            const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
            const float w = ok ? a.weights[s] : 0.f;
            const float m = (ts + te) * 0.5f;
            const float r = (ok && want_near) ? a.d_weights[s] : 0.f;
            const float Ri = cr + (lw_excl_suffix(r, lane) + r);
            const float Wx = cw + lw_excl_suffix(w, lane), WMx = cwm + lw_excl_suffix(w * m, lane);
            cr = __shfl_sync(0xffffffffu, Ri, 0);
            cw = __shfl_sync(0xffffffffu, Wx + w, 0);
            cwm = __shfl_sync(0xffffffffu, WMx + w * m, 0);
            if (ok) {
                float dw = 0.f;
                if (want_near) dw += cn * Ri;
                if (sel) dw += cd * (2.0f * (WMx - m * Wx));
                a.d_weights[s] = dw;
            }
        }
    }
    // pass 3, front to back: empty  ce * w;  dist  cd * (2/3 dt w + 2 sum_{i < k} w_i (m_k - m_i))
    float cw = 0.f, cwm = 0.f;   // prefix sums of the earlier chunks
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
        const float w = ok ? a.weights[s] : 0.f;
        const float m = (ts + te) * 0.5f;
        const float Wpre = cw + lw_excl_scan(w, lane), WMpre = cwm + lw_excl_scan(w * m, lane);
        cw = __shfl_sync(0xffffffffu, Wpre + w, 31);
        cwm = __shfl_sync(0xffffffffu, WMpre + w * m, 31);
        if (ok) {
            float dw = (want_near || sel) ? a.d_weights[s] : 0.f;
            if (want_empty && m < tgt - a.eps_depth) dw += ce * w;
            if (sel) dw += cd * ((2.0f / 3.0f) * (te - ts) * w + 2.0f * (m * Wpre - WMpre));
            a.d_weights[s] = dw;
        }
    }
}

}  // namespace nsb

using namespace nsb;

static int loss_check(const nsb_loss_args *a, const char *who) {
    if (!a || !a->packed_info || !a->t_starts || !a->t_ends || !a->weights || !a->rgb || !a->acc || !a->depth || !a->image ||
        !a->accum || !a->values || !a->coef) {
        set_error("%s: null argument", who);
        return 1;
    }
    return 0;
}

extern "C" int nsb_losses_forward(const nsb_loss_args *args, void *stream) {
    if (loss_check(args, "nsb_losses_forward")) return 1;
    if (args->n_rays <= 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(args->accum, 0, sizeof(double) * A_COUNT, st);
    if (e != cudaSuccess) { set_error("nsb_losses_forward: memset: %s", cudaGetErrorString(e)); return 1; }
    LossK K; K.a = *args;
    losses_fwd_kernel<<<(int)((args->n_rays + 7) / 8), 256, 0, st>>>(K);
    losses_finalize_kernel<<<1, 32, 0, st>>>(K);
    return check_launch("losses_fwd_kernel");
}

extern "C" int nsb_losses_backward(const nsb_loss_args *args, void *stream) {
    if (loss_check(args, "nsb_losses_backward")) return 1;
    if (!args->upstream || !args->d_rgb || !args->d_acc || !args->d_depth || !args->d_weights) { set_error("nsb_losses_backward: gradient buffers missing"); return 1; }
    if (args->n_rays <= 0) return 0;
    LossK K; K.a = *args;
    losses_bwd_kernel<<<(int)((args->n_rays + 7) / 8), 256, 0, (cudaStream_t)stream>>>(K);
    return check_launch("losses_bwd_kernel");
}
