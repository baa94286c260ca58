// Ray marching, visibility filter and alpha compositing for sm_90a.
//
// Replaces (reference, relative to /root/reference/src/nersemble/nerfstudio/):
//   nerfacc OccGridEstimator.sampling -> traverse_grids   (model_components/nersemble_volumetric_sampler.py:95-108)
//   nerfacc render_visibility_from_density                (training pre-pass of sampling())
//   nerfacc pack_info / render_weight_from_density + RGB/Depth/Accumulation renderers
//                                                         (models/nersemble_instant_ngp.py:325-343)
//   DeformationRenderer                                   (model_components/nersemble_deformation_renderer.py:10-29)
//
// The marcher keeps nerfacc's arithmetic order in float32 WITHOUT fused multiply-add
// (__fmul_rn/__fadd_rn) so that sample positions are bit-exact to the CPU oracle
// (oracle/tp/nerfacc_cpu.py): t advances by repeated float32 addition, exactly like
// `t_last = t_last + dt` in nerfacc's traverse_grids kernel.
#include <algorithm>

#include "nsb_common.cuh"
#include "nsb_march.cuh"

namespace nsb {

// ---------------------------------------------------------------------------------------------
// fixed-stride marcher (BASELINE configs 1/2; SURVEY 8d): n_per_ray steps from max(t_enter, near)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) march_fixed_kernel(const float *__restrict__ origins, const float *__restrict__ directions,
                                                          int64_t n_rays, const float *__restrict__ aabb, int n_per_ray, float step,
                                                          float near_plane, float *__restrict__ t_starts, float *__restrict__ t_ends,
                                                          int32_t *__restrict__ ray_indices, int64_t *__restrict__ packed_info) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // one warp per ray
    if (r >= n_rays) return;
    const float t0 = march_fixed_t0(origins, directions, aabb, r, near_plane);
    march_fixed_warp(t0, r, n_per_ray, step, t_starts, t_ends, ray_indices, lane);
    if (packed_info && lane == 0) {
        packed_info[2 * r] = r * n_per_ray;
        packed_info[2 * r + 1] = n_per_ray;
    }
}

// ---------------------------------------------------------------------------------------------
// occupancy-grid marcher: nerfacc csrc/grid.cu traverse_grids (one thread per ray), two passes
// ---------------------------------------------------------------------------------------------
struct MarchArgs {
    nsb_march_args a;
};


template <bool FILL, int LV>
__global__ void __launch_bounds__(128) march_occ_kernel(const __grid_constant__ MarchArgs M) {
    const nsb_march_args &a = M.a;
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n_rays) return;
    const int32_t count = march_occ_ray<FILL, LV>(a, r, FILL ? a.offsets[r] : 0, INT64_MAX);
    if (!FILL) a.counts[r] = count;
}

// ---------------------------------------------------------------------------------------------
// visibility mask (nerfacc render_visibility_from_density): one warp per ray
// ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) visibility_kernel(const int64_t *__restrict__ packed_info, int64_t n_rays,
                                                         const float *__restrict__ t_starts,
                                                         const float *__restrict__ t_ends,
                                                         const float *__restrict__ sigma, float early_stop_eps,
                                                         float alpha_thre, uint8_t *__restrict__ mask,
                                                         int32_t *__restrict__ kept) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    const int64_t start = packed_info[2 * ray], cnt = packed_info[2 * ray + 1];
    float carry = 0.f;
    int32_t k = 0;
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        float sd = 0.f;
        if (i < cnt) sd = sigma[start + i] * (t_ends[start + i] - t_starts[start + i]);
        const float incl = warp_incl_scan(sd, lane);
        const float excl = carry + (incl - sd);
        const float T = expf(-excl);
        const float alpha = 1.0f - expf(-sd);
        bool vis = T >= early_stop_eps;
        if (alpha_thre > 0.0f) vis = vis && (alpha >= alpha_thre);
        if (i < cnt) mask[start + i] = vis ? 1 : 0;
        k += __popc(__ballot_sync(0xffffffffu, vis && i < cnt));
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0 && kept) kept[ray] = k;
}

// ---------------------------------------------------------------------------------------------
// compositing: one warp per ray
// ---------------------------------------------------------------------------------------------
struct CompArgs {
    nsb_composite_args a;
};


__global__ void __launch_bounds__(256) composite_kernel(const __grid_constant__ CompArgs C) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= C.a.n_rays) return;
    composite_ray(C.a, ray, lane);
}

// ---------------------------------------------------------------------------------------------
// compositing backward (training mode): one warp per ray, three passes over the ray's samples.
//   w_i = T_i a_i, T_i = exp(-sum_{j<i} sd_j), a_i = 1-exp(-sd_i), sd = sigma*dt
//   dL/dsd_i = G_i T_i (1-a_i) - sum_{j>i} G_j w_j,  G_i = dL/dw_i (all consumers of w_i)
// The suffix sum_{j>i} G_j w_j is a reverse scan (last chunk first), not total - inclusive prefix: behind an opaque
// surface every later G_j w_j is exactly 0, and so is the suffix, where the subtraction leaves ~eps * |total| of noise.
// ---------------------------------------------------------------------------------------------
struct CompBwdArgs {
    nsb_composite_bwd_args a;
};

// exclusive reverse scan within the warp: sum of v over the lanes above this one
__device__ __forceinline__ float warp_excl_suffix(float v, int lane) {
    float x = __shfl_down_sync(0xffffffffu, v, 1);
    if (lane == 31) x = 0.f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_down_sync(0xffffffffu, x, o);
        if (lane + o < 32) x += t;
    }
    return x;
}

__global__ void __launch_bounds__(256) composite_bwd_kernel(const __grid_constant__ CompBwdArgs C) {
    const nsb_composite_bwd_args &a = C.a;
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
    if (cnt == 0) return;
    const float gr = a.d_out_rgb[3 * ray], gg = a.d_out_rgb[3 * ray + 1], gb = a.d_out_rgb[3 * ray + 2];
    const float gacc = a.d_out_acc ? a.d_out_acc[ray] : 0.f;
    float gdep = a.d_out_depth ? a.d_out_depth[ray] : 0.f;
    // pass 1: forward recompute of acc, N = sum w*mid, and of total = sum_j G_j w_j (needs acc, N first -> split)
    float carry = 0.f, acc = 0.f, N = 0.f;
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
        const float sd = ok ? a.sigma[s] * (te - ts) : 0.f;
        const float incl = warp_incl_scan(sd, lane);
        const float w = ok ? expf(-(carry + (incl - sd))) * (1.0f - expf(-sd)) : 0.f;
        carry += __shfl_sync(0xffffffffu, incl, 31);
        acc += w;
        N += w * ((ts + te) / 2.0f);
    }
    acc = warp_sum(acc);
    N = warp_sum(N);
    const float inv = 1.0f / (acc + 1e-10f);
    const float draw = N * inv;
    if (a.workspace[0] != 0xffffffffu) {   // torch.clip backward: gradient only inside [min, max]
        const float lo = ordered_to_float(a.workspace[0]), hi = ordered_to_float(a.workspace[1]);
        if (!(draw >= lo && draw <= hi)) gdep = 0.f;
    }
    const float gbg = -(gr + gg + gb);     // white background: rgb + (1 - acc)
    // pass 2, front to back: the per-sample terms.  Each sample's G T e, G w, w and dt are parked in its own output slots
    // (d_sigma, d_rgb[0..2]); pass 3 reads them back in the same thread, so no other memory is needed.
    carry = 0.f;
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
        const float dt = te - ts;
        const float sd = ok ? a.sigma[s] * dt : 0.f;
        const float incl = warp_incl_scan(sd, lane);
        const float T = expf(-(carry + (incl - sd)));
        const float e = expf(-sd);
        const float w = ok ? T * (1.0f - e) : 0.f;
        carry += __shfl_sync(0xffffffffu, incl, 31);
        if (ok) {
            const float G = (a.d_weights ? a.d_weights[s] : 0.f) + gr * a.rgb[3 * s] + gg * a.rgb[3 * s + 1] +
                            gb * a.rgb[3 * s + 2] + gbg + gacc + gdep * (((ts + te) / 2.0f) - draw) * inv;
            a.d_sigma[s] = G * T * e;
            a.d_rgb[3 * s] = G * w; a.d_rgb[3 * s + 1] = w; a.d_rgb[3 * s + 2] = dt;
        }
    }
    // pass 3, back to front: suffix = sum_{j>i} G_j w_j as a reverse scan with a carried suffix of the later chunks
    float scarry = 0.f;
    for (int64_t b = ((cnt - 1) >> 5) << 5; b >= 0; b -= 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float gte = ok ? a.d_sigma[s] : 0.f, gw = ok ? a.d_rgb[3 * s] : 0.f;
        const float w = ok ? a.d_rgb[3 * s + 1] : 0.f, dt = ok ? a.d_rgb[3 * s + 2] : 0.f;
        const float suffix = scarry + warp_excl_suffix(gw, lane);
        scarry = __shfl_sync(0xffffffffu, suffix + gw, 0);
        if (ok) {
            a.d_sigma[s] = (gte - suffix) * dt;
            a.d_rgb[3 * s] = gr * w; a.d_rgb[3 * s + 1] = gg * w; a.d_rgb[3 * s + 2] = gb * w;
        }
    }
}

__global__ void depth_init_kernel(uint32_t *ws) {
    ws[0] = 0xffffffffu;
    ws[1] = 0u;
}

// DepthRenderer('expected'): depth = clip(depth, steps.min(), steps.max()) over ALL samples of the batch
__global__ void depth_clip_kernel(float *depth, int64_t n_rays, const uint32_t *ws) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    if (ws[0] == 0xffffffffu) return;  // no samples at all
    const float lo = ordered_to_float(ws[0]), hi = ordered_to_float(ws[1]);
    depth[r] = fminf(fmaxf(depth[r], lo), hi);
}

// ---------------------------------------------------------------------------------------------
// occupancy-grid EMA update (nerfacc OccGridEstimator._update): see nsb.h.  occ values are >= 0 (densities), so the
// int ordering of their bit patterns is the float ordering and atomicMax(int) resolves duplicate cells.
// ---------------------------------------------------------------------------------------------
__global__ void occ_decay_kernel(const float *__restrict__ occs, const int64_t *__restrict__ ids, int64_t n, float decay,
                                 float *__restrict__ tmp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tmp[ids[i]] = occs[ids[i]] * decay;      // duplicates store the same value
}
__global__ void occ_max_kernel(const int64_t *__restrict__ ids, const float *__restrict__ occ_new, int64_t n,
                               float *__restrict__ tmp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = occ_new[i];
    if (v >= 0.f) atomicMax(reinterpret_cast<int *>(tmp + ids[i]), __float_as_int(v));
    else if (isnan(v)) tmp[ids[i]] = v;                  // torch.maximum propagates NaN
}
__global__ void occ_commit_kernel(float *__restrict__ occs, const int64_t *__restrict__ ids, int64_t n,
                                  const float *__restrict__ tmp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) occs[ids[i]] = tmp[ids[i]];
}
__global__ void __launch_bounds__(256) occ_mean_kernel(const float *__restrict__ occs, int64_t n_cells, double *__restrict__ acc) {
    double s = 0.0, c = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = occs[i];
        if (v >= 0.f) { s += (double)v; c += 1.0; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    if ((threadIdx.x & 31) == 0 && c > 0.0) { atomicAdd(acc, s); atomicAdd(acc + 1, c); }
}
__global__ void occ_binarise_kernel(const float *__restrict__ occs, int64_t n_cells, const double *__restrict__ acc,
                                    float occ_thre, uint8_t *__restrict__ binaries) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cells) return;
    const float mean = (float)(acc[0] / acc[1]);        // 0/0 = NaN like torch.mean of an empty selection
    const float thre = fminf(mean, occ_thre);            // torch.clamp(mean, max=occ_thre); NaN mean -> occ_thre
    binaries[i] = occs[i] > (isnan(mean) ? occ_thre : thre) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// occupancy march in ONE cooperative launch: samples per ray | grid barrier | per-CTA chunk sums | barrier | exclusive
// scan -> packed_info + total | barrier | fill.  No host synchronisation: the packed count goes to the workspace header
// (nsb_render_ws_header.n_total) where the fused field + composite kernel (render_kernel_ws, sampler GIVEN) reads it.
// ---------------------------------------------------------------------------------------------
struct MarchCoopArgs {
    nsb_march_args M;
    int64_t *packed_info;
    nsb_render_ws_header *hdr;
    int64_t *partials;
    int64_t capacity;
    float *scratch;          // [2][capacity] or NULL: single traversal into per-ray slots, then a packing copy
    int64_t slot;            // capacity / n_rays
};
constexpr int kCoopThreads = 256;

__device__ __forceinline__ void coop_grid_barrier(uint32_t *ctr, const uint32_t target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        uint32_t v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
            if (v < target) __nanosleep(40);
        } while (v < target);
        __threadfence();
    }
    __syncthreads();
}
__device__ __forceinline__ int64_t coop_block_sum(int64_t v, int64_t *red, const int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    int64_t t = 0;
    for (int w = 0; w < kCoopThreads / 32; ++w) t += red[w];
    return t;
}

// Exclusive scan of per-ray counts -> packed_info (start, count), total -> hdr->n_total, across a cooperative grid:
// per-CTA chunk sums | grid barrier (index first_barrier + 1) | chunk bases + in-chunk slab scans.  The caller puts a
// barrier after it.  status = total > capacity, or a pre-set hdr->reserved[0] (a truncated ray); beyond the capacity
// rays are truncated so that nothing downstream reads or writes out of bounds.
__device__ __forceinline__ void coop_scan_counts(const int32_t *counts, const int64_t R, int64_t *packed_info, int64_t *partials,
                                                 nsb_render_ws_header *hdr, const int64_t capacity, int64_t *red,
                                                 const uint32_t first_barrier) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t chunk = (R + gridDim.x - 1) / gridDim.x;
    const int64_t r0 = min(R, (int64_t)blockIdx.x * chunk), r1 = min(R, r0 + chunk);
    {
        int64_t v = 0;
        for (int64_t r = r0 + tid; r < r1; r += kCoopThreads) v += __ldcg(counts + r);
        const int64_t tot = coop_block_sum(v, red, tid);
        if (tid == 0) partials[blockIdx.x] = tot;
    }
    coop_grid_barrier(&hdr->barrier, (first_barrier + 1u) * gridDim.x);
    int64_t before = 0, total = 0;
    for (int b = tid; b < (int)gridDim.x; b += kCoopThreads) {
        const int64_t p = __ldcg(partials + b);
        total += p;
        if (b < (int)blockIdx.x) before += p;
    }
    total = coop_block_sum(total, red, tid);
    before = coop_block_sum(before, red, tid);
    if (blockIdx.x == 0 && tid == 0) {
        hdr->n_total = total;
        hdr->status = (total > capacity || __ldcg(&hdr->reserved[0]) != 0) ? 1 : 0;
    }
    int64_t carry = before;
    for (int64_t s0 = r0; s0 < r1; s0 += kCoopThreads) {
        const int64_t r = s0 + tid;
        const int64_t c = r < r1 ? (int64_t)__ldcg(counts + r) : 0;
        int64_t inc = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t nb = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += nb;
        }
        __syncthreads();
        if (lane == 31) red[warp] = inc;
        __syncthreads();
        int64_t wbase = 0, slab = 0;
        for (int w = 0; w < kCoopThreads / 32; ++w) {
            const int64_t t = red[w];
            if (w < warp) wbase += t;
            slab += t;
        }
        if (r < r1) {
            const int64_t st = min(carry + wbase + inc - c, capacity);
            packed_info[2 * r] = st;
            packed_info[2 * r + 1] = min(c, capacity - st);
        }
        carry += slab;
    }
}

template <int LV>
__global__ void __launch_bounds__(kCoopThreads) march_occ_coop_kernel(const __grid_constant__ MarchCoopArgs K) {
    __shared__ int64_t red[kCoopThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t R = K.M.n_rays;
    uint32_t *const bar = &K.hdr->barrier;
    const bool single = K.scratch != nullptr;
    if (single) {
        // ONE traversal: the samples of ray r go to its slot [r * slot, (r + 1) * slot) of the scratch arrays
        MarchArgs S1; S1.a = K.M;
        S1.a.t_starts = K.scratch; S1.a.t_ends = K.scratch + K.capacity; S1.a.ray_indices = nullptr;
        bool over = false;
        // rays are dealt round-robin to the CTAs (ray = block + grid * k): a thread per ray writes 2 scattered words per
        // sample, and with consecutive rays per CTA 4096 rays kept the store pipes of 16 SMs busy while 132 SMs idled
        for (int64_t r = (int64_t)blockIdx.x + (int64_t)gridDim.x * tid; r < R; r += (int64_t)gridDim.x * kCoopThreads) {
            const int32_t c = march_occ_ray<true, LV>(S1.a, r, r * K.slot, (r + 1) * K.slot);
            over |= c > K.slot;
            K.M.counts[r] = (int32_t)min((int64_t)c, K.slot);
        }
        if (over) K.hdr->reserved[0] = 1;                 // folded into status by block 0 after the barrier
    } else {
        for (int64_t r = (int64_t)blockIdx.x + (int64_t)gridDim.x * tid; r < R; r += (int64_t)gridDim.x * kCoopThreads)
            K.M.counts[r] = march_occ_ray<false, LV>(K.M, r, 0, 0);
    }
    coop_grid_barrier(bar, 1u * gridDim.x);
    coop_scan_counts(K.M.counts, R, K.packed_info, K.partials, K.hdr, K.capacity, red, 1u);
    coop_grid_barrier(bar, 3u * gridDim.x);
    if (single) {
        // packing copy, one warp per ray: coalesced reads of the slot, coalesced writes of the packed arrays
        const float *s_ts = K.scratch, *s_te = K.scratch + K.capacity;
        for (int64_t r = (int64_t)blockIdx.x * (kCoopThreads / 32) + warp; r < R; r += (int64_t)gridDim.x * (kCoopThreads / 32)) {
            const int64_t dst = __ldcg(K.packed_info + 2 * r), cnt = __ldcg(K.packed_info + 2 * r + 1), src = r * K.slot;
            for (int64_t k = lane; k < cnt; k += 32) {
                K.M.t_starts[dst + k] = __ldcg(s_ts + src + k);
                K.M.t_ends[dst + k] = __ldcg(s_te + src + k);
                K.M.ray_indices[dst + k] = (int32_t)r;
            }
        }
    } else {
        for (int64_t r = (int64_t)blockIdx.x + (int64_t)gridDim.x * tid; r < R; r += (int64_t)gridDim.x * kCoopThreads)
            march_occ_ray<true, LV>(K.M, r, __ldcg(K.packed_info + 2 * r), K.capacity);
    }
}

// grid of a cooperative launch of Kernel: every CTA resident, at most 4 per SM and at most 1024 (the scan partials)
template <auto Kernel>
static int coop_grid() {
    static int grid = 0;
    if (grid == 0) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, Kernel, kCoopThreads, 0);
        grid = std::max(1, std::min(sms * std::max(1, std::min(per_sm, 4)), 1024));
    }
    return grid;
}

int launch_march_occ_coop(const nsb_march_args &M, int64_t *packed_info, nsb_render_ws_header *hdr, int64_t *partials,
                          int64_t capacity, float *scratch, cudaStream_t st) {
    MarchCoopArgs K;
    K.M = M; K.packed_info = packed_info; K.hdr = hdr; K.partials = partials; K.capacity = capacity;
    K.slot = capacity / std::max<int64_t>(M.n_rays, 1);
    K.scratch = K.slot >= 1 ? scratch : nullptr;
    const int grid = coop_grid<march_occ_coop_kernel<1>>();
    cudaError_t e = cudaMemsetAsync(hdr, 0, sizeof(nsb_render_ws_header), st);      // barrier, status, reserved[0]
    if (e != cudaSuccess) { set_error("march_occ_coop: memset: %s", cudaGetErrorString(e)); return 2; }
    void *kargs[] = {&K};
    const void *fn = M.levels == 1 ? reinterpret_cast<const void *>(march_occ_coop_kernel<1>)
                                   : reinterpret_cast<const void *>(march_occ_coop_kernel<0>);
    e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kCoopThreads), kargs, 0, st);
    if (e != cudaSuccess) { set_error("march_occ_coop_kernel: %s", cudaGetErrorString(e)); return 2; }
    return check_launch("march_occ_coop_kernel");
}

// ---------------------------------------------------------------------------------------------
// visibility filter + compaction of the kept samples in ONE cooperative launch (sync-free training sampler):
//   V1 warp per ray: nerfacc render_visibility_from_density (same arithmetic as visibility_kernel), mask bytes + kept count
//   V2 exclusive scan of the kept counts -> out_packed_info, total -> header.n_total
//   V3 warp per ray: ballot-compaction of t_starts / t_ends / ray_indices and of the optional payload rows
// ---------------------------------------------------------------------------------------------
struct VisCompactK {
    nsb_vis_compact_args a;
    nsb_render_ws_header *hdr;
    int64_t *partials;
    int32_t *counts;
    uint8_t *mask;
};

__global__ void __launch_bounds__(kCoopThreads) vis_compact_coop_kernel(const __grid_constant__ VisCompactK K) {
    __shared__ int64_t red[kCoopThreads / 32];
    const nsb_vis_compact_args &a = K.a;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t R = a.n_rays;
    float alpha_thre = a.alpha_thre;
    if (a.alpha_thre_cap) alpha_thre = fminf(alpha_thre, __ldg(a.alpha_thre_cap));   // min(alpha_thre, occs.mean())
    for (int64_t ray = (int64_t)blockIdx.x * (kCoopThreads / 32) + warp; ray < R; ray += (int64_t)gridDim.x * (kCoopThreads / 32)) {
        const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
        float carry = 0.f;
        int32_t k = 0;
        for (int64_t b = 0; b < cnt; b += 32) {
            const int64_t i = b + lane;
            float sd = 0.f;
            if (i < cnt) sd = a.sigma[start + i] * (a.t_ends[start + i] - a.t_starts[start + i]);
            const float incl = warp_incl_scan(sd, lane);
            const float excl = carry + (incl - sd);
            const float T = expf(-excl);
            const float alpha = 1.0f - expf(-sd);
            bool vis = T >= a.early_stop_eps;
            if (alpha_thre > 0.0f) vis = vis && (alpha >= alpha_thre);
            if (i < cnt) K.mask[start + i] = vis ? 1 : 0;
            k += __popc(__ballot_sync(0xffffffffu, vis && i < cnt));
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) K.counts[ray] = k;
    }
    coop_grid_barrier(&K.hdr->barrier, 1u * gridDim.x);
    coop_scan_counts(K.counts, R, a.out_packed_info, K.partials, K.hdr, a.capacity, red, 1u);
    coop_grid_barrier(&K.hdr->barrier, 3u * gridDim.x);
    for (int64_t ray = (int64_t)blockIdx.x * (kCoopThreads / 32) + warp; ray < R; ray += (int64_t)gridDim.x * (kCoopThreads / 32)) {
        const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
        int64_t dst = __ldcg(a.out_packed_info + 2 * ray);
        for (int64_t b = 0; b < cnt; b += 32) {
            const int64_t i = b + lane;
            const bool keep = i < cnt && K.mask[start + i] != 0;
            const uint32_t bal = __ballot_sync(0xffffffffu, keep);
            const int64_t pos = dst + __popc(bal & ((1u << lane) - 1u));
            if (keep) {
                a.out_t_starts[pos] = a.t_starts[start + i];
                a.out_t_ends[pos] = a.t_ends[start + i];
                a.out_ray_indices[pos] = a.ray_indices[start + i];
                if (a.xs) reinterpret_cast<float4 *>(a.out_xs)[pos] = reinterpret_cast<const float4 *>(a.xs)[start + i];
            }
            if (a.feat || a.corner_vals) {      // payload rows: the warp moves one kept sample at a time, 16 B per lane
                uint32_t m = bal;
                int64_t p = dst;
                while (m) {
                    const int src_lane = __ffs(m) - 1;
                    m &= m - 1;
                    const int64_t si = start + b + src_lane;
                    if (a.corner_vals)
                        reinterpret_cast<uint4 *>(a.out_corner_vals)[p * 32 + lane] = reinterpret_cast<const uint4 *>(a.corner_vals)[si * 32 + lane];
                    if (a.feat && lane < 4)
                        reinterpret_cast<uint4 *>(a.out_feat)[p * 4 + lane] = reinterpret_cast<const uint4 *>(a.feat)[si * 4 + lane];
                    ++p;
                }
            }
            dst += __popc(bal);
        }
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_march_fixed(const float *origins, const float *directions, int64_t n_rays, const float *aabb6,
                               int32_t n_per_ray, float step, float near_plane, float *t_starts, float *t_ends,
                               int32_t *ray_indices, int64_t *packed_info, void *stream) {
    if (!origins || !directions || !aabb6 || !t_starts || !t_ends || !ray_indices) {
        set_error("nsb_march_fixed: null argument");
        return 1;
    }
    if (n_rays <= 0 || n_per_ray <= 0) return 0;
    const int threads = 256;
    const int blocks = (int)((n_rays + 7) / 8);
    march_fixed_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(origins, directions, n_rays, aabb6, n_per_ray, step,
                                                                   near_plane, t_starts, t_ends, ray_indices, packed_info);
    return check_launch("march_fixed_kernel");
}

extern "C" int nsb_march_occupancy(const nsb_march_args *args, void *stream) {
    if (!args || !args->origins || !args->directions || !args->near_planes || !args->far_planes || !args->binaries ||
        !args->aabbs) {
        set_error("nsb_march_occupancy: null argument");
        return 1;
    }
    if (args->levels < 1 || args->levels > 8) { set_error("nsb_march_occupancy: levels must be in [1,8]"); return 1; }
    if (args->n_rays <= 0) return 0;
    MarchArgs M; M.a = *args;
    const int threads = 128;
    const int blocks = (int)((args->n_rays + threads - 1) / threads);
    if (args->t_starts == nullptr) {
        if (!args->counts) { set_error("nsb_march_occupancy: pass 1 needs counts"); return 1; }
        if (args->levels == 1) march_occ_kernel<false, 1><<<blocks, threads, 0, (cudaStream_t)stream>>>(M);
        else march_occ_kernel<false, 0><<<blocks, threads, 0, (cudaStream_t)stream>>>(M);
    } else {
        if (!args->offsets || !args->t_ends || !args->ray_indices) { set_error("nsb_march_occupancy: pass 2 needs offsets/t_ends/ray_indices"); return 1; }
        if (args->levels == 1) march_occ_kernel<true, 1><<<blocks, threads, 0, (cudaStream_t)stream>>>(M);
        else march_occ_kernel<true, 0><<<blocks, threads, 0, (cudaStream_t)stream>>>(M);
    }
    return check_launch("march_occ_kernel");
}

extern "C" int nsb_visibility_mask(const int64_t *packed_info, int64_t n_rays, const float *t_starts,
                                   const float *t_ends, const float *sigma, float early_stop_eps, float alpha_thre,
                                   uint8_t *mask, int32_t *kept_counts, void *stream) {
    if (!packed_info || !t_starts || !t_ends || !sigma || !mask) { set_error("nsb_visibility_mask: null argument"); return 1; }
    if (n_rays <= 0) return 0;
    const int blocks = (int)((n_rays + 7) / 8);
    visibility_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(packed_info, n_rays, t_starts, t_ends, sigma,
                                                              early_stop_eps, alpha_thre, mask, kept_counts);
    return check_launch("visibility_kernel");
}

extern "C" int nsb_composite_backward(const nsb_composite_bwd_args *args, void *stream) {
    if (!args || !args->packed_info || !args->t_starts || !args->t_ends || !args->sigma || !args->rgb || !args->d_out_rgb ||
        !args->workspace || !args->d_sigma || !args->d_rgb) {
        set_error("nsb_composite_backward: null argument");
        return 1;
    }
    if (args->n_rays <= 0) return 0;
    CompBwdArgs C; C.a = *args;
    const int blocks = (int)((args->n_rays + 7) / 8);
    composite_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(C);
    return check_launch("composite_bwd_kernel");
}

extern "C" int nsb_composite_forward(const nsb_composite_args *args, void *stream) {
    if (!args || !args->packed_info || !args->t_starts || !args->t_ends || !args->sigma || !args->rgb || !args->out_rgb ||
        !args->out_acc || !args->out_depth || !args->workspace) {
        set_error("nsb_composite_forward: null argument");
        return 1;
    }
    if (args->n_rays <= 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    CompArgs C; C.a = *args;
    depth_init_kernel<<<1, 1, 0, st>>>(args->workspace);
    const int blocks = (int)((args->n_rays + 7) / 8);
    composite_kernel<<<blocks, 256, 0, st>>>(C);
    depth_clip_kernel<<<(int)((args->n_rays + 255) / 256), 256, 0, st>>>(args->out_depth, args->n_rays, args->workspace);
    return check_launch("composite_kernel");
}

extern "C" size_t nsb_occ_update_scratch_bytes(int64_t n_cells) { return (size_t)n_cells * sizeof(float) + 2 * sizeof(double) + 8; }

extern "C" int nsb_occ_update(float *occs, uint8_t *binaries, int64_t n_cells, const int64_t *cell_ids, const float *occ_new,
                              int64_t n, float ema_decay, float occ_thre, void *scratch, void *stream) {
    if (!occs || !binaries || !scratch || n_cells <= 0 || (n > 0 && (!cell_ids || !occ_new))) {
        set_error("nsb_occ_update: null argument");
        return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double *acc = reinterpret_cast<double *>(scratch);                                   // 8-byte aligned head
    float *tmp = reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(scratch) + 2 * sizeof(double));
    const int T = 256;
    if (n > 0) {
        const int blocks = (int)((n + T - 1) / T);
        occ_decay_kernel<<<blocks, T, 0, st>>>(occs, cell_ids, n, ema_decay, tmp);
        occ_max_kernel<<<blocks, T, 0, st>>>(cell_ids, occ_new, n, tmp);
        occ_commit_kernel<<<blocks, T, 0, st>>>(occs, cell_ids, n, tmp);
    }
    cudaMemsetAsync(acc, 0, 2 * sizeof(double), st);
    occ_mean_kernel<<<296, 256, 0, st>>>(occs, n_cells, acc);
    occ_binarise_kernel<<<(int)((n_cells + T - 1) / T), T, 0, st>>>(occs, n_cells, acc, occ_thre, binaries);
    return check_launch("nsb_occ_update");
}

extern "C" int nsb_march_occupancy_packed(const nsb_march_args *args, int64_t capacity, int64_t *packed_info, void *workspace,
                                          float *scratch, void *stream) {
    if (!args || !args->origins || !args->directions || !args->near_planes || !args->far_planes || !args->binaries ||
        !args->aabbs || !args->t_starts || !args->t_ends || !args->ray_indices || !packed_info || !workspace) {
        set_error("nsb_march_occupancy_packed: null argument");
        return 1;
    }
    if (args->levels < 1 || args->levels > 8 || capacity <= 0) { set_error("nsb_march_occupancy_packed: levels must be in [1,8], capacity > 0"); return 1; }
    if (args->n_rays <= 0) return 0;
    uint8_t *ws = reinterpret_cast<uint8_t *>(workspace);
    nsb_march_args M = *args;
    M.counts = reinterpret_cast<int32_t *>(ws + 64 + 1024 * sizeof(int64_t));
    M.offsets = nullptr;
    return launch_march_occ_coop(M, packed_info, reinterpret_cast<nsb_render_ws_header *>(ws), reinterpret_cast<int64_t *>(ws + 64),
                                 capacity, scratch, (cudaStream_t)stream);
}

extern "C" int nsb_visibility_compact(const nsb_vis_compact_args *args, void *stream) {
    if (!args || !args->packed_info || !args->t_starts || !args->t_ends || !args->sigma || !args->ray_indices ||
        !args->out_packed_info || !args->out_t_starts || !args->out_t_ends || !args->out_ray_indices || !args->workspace) {
        set_error("nsb_visibility_compact: null argument");
        return 1;
    }
    if ((args->feat && !args->out_feat) || (args->xs && !args->out_xs) || (args->corner_vals && !args->out_corner_vals)) {
        set_error("nsb_visibility_compact: payload without destination");
        return 1;
    }
    if (args->n_rays <= 0) return 0;
    uint8_t *ws = reinterpret_cast<uint8_t *>(args->workspace);
    VisCompactK K;
    K.a = *args;
    K.hdr = reinterpret_cast<nsb_render_ws_header *>(ws);
    K.partials = reinterpret_cast<int64_t *>(ws + 64);
    K.counts = reinterpret_cast<int32_t *>(ws + 64 + 1024 * sizeof(int64_t));
    // mask bytes: behind the counts (the workspace of nsb_vis_compact_workspace_bytes)
    K.mask = ws + 64 + 1024 * sizeof(int64_t) + (((size_t)args->n_rays * sizeof(int32_t) + 63) / 64) * 64;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = coop_grid<vis_compact_coop_kernel>();
    cudaError_t e = cudaMemsetAsync(K.hdr, 0, sizeof(nsb_render_ws_header), st);
    if (e != cudaSuccess) { set_error("nsb_visibility_compact: memset: %s", cudaGetErrorString(e)); return 2; }
    void *kargs[] = {&K};
    e = cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(vis_compact_coop_kernel), dim3(grid), dim3(kCoopThreads), kargs, 0, st);
    if (e != cudaSuccess) { set_error("vis_compact_coop_kernel: %s", cudaGetErrorString(e)); return 2; }
    return check_launch("vis_compact_coop_kernel");
}

extern "C" size_t nsb_vis_compact_workspace_bytes(int64_t n_rays, int64_t capacity) {
    return 64 + 1024 * sizeof(int64_t) + (((size_t)std::max<int64_t>(n_rays, 1) * sizeof(int32_t) + 63) / 64) * 64 + (size_t)capacity + 64;
}
