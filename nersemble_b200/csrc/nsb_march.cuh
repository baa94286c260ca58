// Per-ray device code of the marchers and the compositor, shared by the stand-alone kernels (nsb_render.cu) and the
// fused render kernel (nsb_field.cu): both paths run the SAME arithmetic, so their results are bit-identical.
#pragma once
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ float calc_dt(float t, float cone_angle, float dt_min, float dt_max) {
    return fminf(fmaxf(__fmul_rn(t, cone_angle), dt_min), dt_max);
}

__device__ __forceinline__ float warp_incl_scan(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One ray of nerfacc's traverse_grids (csrc/grid.cu, one thread per ray).  FILL = false: returns the sample count.
// FILL = true: writes the samples at out_base.. (only below out_limit: the capacity guard of the fused render kernel).
// LV = 0: a.levels grids (<= 8, the interval arrays are indexed dynamically and live in local memory); LV = 1: the
// single-level specialisation of the NeRSemble recipe (grid_levels = 1, train_nersemble.py:102): everything in registers.
template <bool FILL, int LV = 0>
__device__ __forceinline__ int32_t march_occ_ray(const nsb_march_args &a, const int64_t r, const int64_t out_base,
                                                 const int64_t out_limit) {
    const float o[3] = {a.origins[3 * r], a.origins[3 * r + 1], a.origins[3 * r + 2]};
    const float d[3] = {a.directions[3 * r], a.directions[3 * r + 1], a.directions[3 * r + 2]};
    const float near_plane = a.near_planes[r], far_plane = a.far_planes[r];
    const float step = a.step, cone = a.cone_angle;
    if (!(isfinite(o[0]) && isfinite(o[1]) && isfinite(o[2]) && isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2])) ||
        (d[0] == 0.f && d[1] == 0.f && d[2] == 0.f)) {
        return 0;   // degenerate ray: no samples (never hang)
    }
    const int res = a.res, levels = LV ? LV : a.levels;
    const float eps = 1e-6f;
    float inv_d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) inv_d[k] = __fdiv_rn(1.0f, d[k]);

    // sorted aabb intersections over levels (tiny insertion sort, stable like torch.sort on ties)
    constexpr int kMaxLevels = LV ? LV : 8;
    float tv[2 * kMaxLevels];
    int ti[2 * kMaxLevels];
    bool hits[kMaxLevels];
#pragma unroll
    for (int lv = 0; lv < levels; ++lv) {
        float t0, t1;
        bool h = ray_aabb(o, d, a.aabbs + 6 * lv, t0, t1);
        hits[lv] = h;
        tv[lv] = h ? t0 : INFINITY;
        tv[levels + lv] = h ? t1 : INFINITY;
        ti[lv] = lv;
        ti[levels + lv] = levels + lv;
    }
#pragma unroll
    for (int i = 1; i < 2 * levels; ++i) {
        float v = tv[i]; int id = ti[i]; int j = i - 1;
        while (j >= 0 && tv[j] > v) { tv[j + 1] = tv[j]; ti[j + 1] = ti[j]; --j; }
        tv[j + 1] = v; ti[j + 1] = id;
    }

    int64_t out = out_base;
    int32_t count = 0;
    float t_last = near_plane;
    bool continuous = false;
    const float resf = (float)res;
#pragma unroll
    for (int i = 0; i < 2 * levels - 1; ++i) {
        const int level = ti[i] % levels;
        if (!hits[level]) continue;
        const float this_tmin = fmaxf(tv[i], near_plane);
        const float this_tmax = fminf(tv[i + 1], far_plane);
        if (!(this_tmin < this_tmax)) continue;
        if (!continuous) {
            if (step <= 0.0f) {
                t_last = this_tmin;
            } else {
                while (true) {
                    const float dt = calc_dt(t_last, cone, step, 1e10f);
                    if (__fadd_rn(t_last, __fmul_rn(dt, 0.5f)) >= this_tmin) break;
                    t_last = __fadd_rn(t_last, dt);
                }
            }
        }
        const float *ab = a.aabbs + 6 * level;
        float tdist[3], delta[3];
        int cur[3], fin[3], stp[3];
        const float ts_eps = __fadd_rn(this_tmin, eps), te_eps = __fsub_rn(this_tmax, eps);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float ext = __fsub_rn(ab[3 + k], ab[k]);
            const float voxel = __fdiv_rn(ext, resf);
            const float rs = __fadd_rn(o[k], __fmul_rn(d[k], ts_eps));
            const float re = __fadd_rn(o[k], __fmul_rn(d[k], te_eps));
            int c = (int)__fmul_rn(__fdiv_rn(__fsub_rn(rs, ab[k]), ext), resf);
            int f = (int)__fmul_rn(__fdiv_rn(__fsub_rn(re, ab[k]), ext), resf);
            c = min(max(c, 0), res - 1);
            f = min(max(f, 0), res - 1);
            cur[k] = c; fin[k] = f;
            const int start_index = c + (d[k] > 0.0f ? 1 : 0);
            const float tmax_k =
                __fadd_rn(__fmul_rn(__fadd_rn(ab[k], __fsub_rn(__fmul_rn((float)start_index, voxel), rs)), inv_d[k]), this_tmin);
            const float sf = d[k] == 0.0f ? 0.0f : (d[k] > 0.0f ? 1.0f : -1.0f);
            tdist[k] = d[k] == 0.0f ? this_tmax : tmax_k;
            delta[k] = d[k] == 0.0f ? this_tmax : __fmul_rn(__fmul_rn(voxel, inv_d[k]), sf);
            stp[k] = (int)sf;
        }
        const int ovf[3] = {fin[0] + stp[0], fin[1] + stp[1], fin[2] + stp[2]};
        // The DDA's cell sequence does not depend on the occupancy bits, so it runs kAhead cells ahead of the sample
        // emission: the kAhead occupancy loads of a group are independent (one L2 round trip per group instead of one
        // per cell -- with 4096 rays = 4096 threads the marcher is pure latency).
        // Cells are processed in the original order with the original arithmetic: bit-identical samples.
        constexpr int kAhead = 4;
        bool finished = false;
        for (int guard = 0; guard < 3 * res + 3 && !finished; guard += kAhead) {
            float tt[kAhead];
            uint32_t cc[kAhead];
            uint8_t oc[kAhead];
            int nv = 0;
#pragma unroll
            for (int j = 0; j < kAhead; ++j) {
                if (!finished && guard + j < 3 * res + 3) {
                    tt[j] = fminf(fminf(tdist[0], fminf(tdist[1], tdist[2])), this_tmax);
                    cc[j] = (uint32_t)((level * res + cur[0]) * res * res + cur[1] * res + cur[2]);   // < 8 * 2^21 cells
                    nv = j + 1;
                    int ax;
                    if (tdist[0] < tdist[1] && tdist[0] < tdist[2]) ax = 0;
                    else if (tdist[1] < tdist[2]) ax = 1;
                    else ax = 2;
                    // (dynamic register-array indexing avoided)
                    bool done;
                    if (ax == 0) { cur[0] += stp[0]; tdist[0] = __fadd_rn(tdist[0], delta[0]); done = cur[0] == ovf[0]; }
                    else if (ax == 1) { cur[1] += stp[1]; tdist[1] = __fadd_rn(tdist[1], delta[1]); done = cur[1] == ovf[1]; }
                    else { cur[2] += stp[2]; tdist[2] = __fadd_rn(tdist[2], delta[2]); done = cur[2] == ovf[2]; }
                    if (done) finished = true;
                } else {
                    tt[j] = 0.f; cc[j] = 0;
                }
            }
#pragma unroll
            for (int j = 0; j < kAhead; ++j) oc[j] = j < nv ? a.binaries[cc[j]] : (uint8_t)0;
#pragma unroll
            for (int j = 0; j < kAhead; ++j) {
                if (j >= nv) break;
                const float t_trav = tt[j];
                if (!oc[j]) {
                    if (step <= 0.0f) {
                        t_last = t_trav;
                    } else {
                        while (true) {
                            const float dt = calc_dt(t_last, cone, step, 1e10f);
                            if (__fadd_rn(t_last, __fmul_rn(dt, 0.5f)) >= t_trav) break;
                            t_last = __fadd_rn(t_last, dt);
                        }
                    }
                    continuous = false;
                } else {
                    while (true) {
                        float t_next;
                        if (step <= 0.0f) {
                            t_next = t_trav;
                        } else {
                            const float dt = calc_dt(t_last, cone, step, 1e10f);
                            if (__fadd_rn(t_last, __fmul_rn(dt, 0.5f)) >= t_trav) break;
                            t_next = __fadd_rn(t_last, dt);
                        }
                        if (FILL) {
                            if (out < out_limit) {
                                a.t_starts[out] = t_last;
                                a.t_ends[out] = t_next;
                                if (a.ray_indices) a.ray_indices[out] = (int32_t)r;
                            }
                            ++out;
                        }
                        ++count;
                        continuous = true;
                        t_last = t_next;
                        if (t_next >= t_trav) break;
                    }
                }
            }
        }
    }
    return count;
}

// One ray of render_weight_from_density + the RGB(white) / expected-depth / accumulation / deformation renderers by one
// warp (lane-strided samples, shuffle scan of sigma*dt).  Shared by composite_kernel and the fused render kernel, so
// the two paths are bit-identical.
__device__ __forceinline__ void composite_ray(const nsb_composite_args &a, const int64_t ray, const int lane) {
    const int64_t start = a.packed_info[2 * ray], cnt = a.packed_info[2 * ray + 1];
    float carry = 0.f;
    float acc = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, dep = 0.f, d0 = 0.f, d1 = 0.f, d2 = 0.f;
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t b = 0; b < cnt; b += 32) {
        const int64_t i = b + lane;
        const bool ok = i < cnt;
        const int64_t s = start + (ok ? i : 0);
        const float ts = ok ? a.t_starts[s] : 0.f, te = ok ? a.t_ends[s] : 0.f;
        const float sd = ok ? a.sigma[s] * (te - ts) : 0.f;
        // render_weight_from_density: T = exp(-exclusive_sum(sigma*dt)), alpha = 1 - exp(-sigma*dt)
        const float incl = warp_incl_scan(sd, lane);
        const float excl = carry + (incl - sd);
        const float w = ok ? expf(-excl) * (1.0f - expf(-sd)) : 0.f;
        carry += __shfl_sync(0xffffffffu, incl, 31);
        if (ok) {
            if (a.out_weights) a.out_weights[s] = w;
            float r = a.rgb[3 * s], g = a.rgb[3 * s + 1], bl = a.rgb[3 * s + 2];
            if (!a.training) {  // RGBRenderer eval path: nan_to_num before compositing
                r = isnan(r) ? 0.f : (isinf(r) ? (r > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f) : r);
                g = isnan(g) ? 0.f : (isinf(g) ? (g > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f) : g);
                bl = isnan(bl) ? 0.f : (isinf(bl) ? (bl > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f) : bl);
            }
            const float mid = (ts + te) / 2.0f;
            acc += w; cr += w * r; cg += w * g; cb += w * bl; dep += w * mid;
            mn = fminf(mn, mid); mx = fmaxf(mx, mid);
            if (a.offsets) { d0 += w * a.offsets[3 * s]; d1 += w * a.offsets[3 * s + 1]; d2 += w * a.offsets[3 * s + 2]; }
        }
    }
    acc = warp_sum(acc); cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb); dep = warp_sum(dep);
    if (a.offsets) { d0 = warp_sum(d0); d1 = warp_sum(d1); d2 = warp_sum(d2); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane == 0) {
        // white background: rgb + 1*(1-acc); eval clamps to [0,1]
        float r = cr + (1.0f - acc), g = cg + (1.0f - acc), bl = cb + (1.0f - acc);
        if (!a.training) { r = fminf(fmaxf(r, 0.f), 1.f); g = fminf(fmaxf(g, 0.f), 1.f); bl = fminf(fmaxf(bl, 0.f), 1.f); }
        a.out_rgb[3 * ray] = r; a.out_rgb[3 * ray + 1] = g; a.out_rgb[3 * ray + 2] = bl;
        a.out_acc[ray] = acc;
        a.out_depth[ray] = dep / (acc + 1e-10f);   // clipped by depth_clip_kernel
        if (a.out_deform) { a.out_deform[3 * ray] = d0; a.out_deform[3 * ray + 1] = d1; a.out_deform[3 * ray + 2] = d2; }
        if (cnt > 0) {
            atomicMin(&a.workspace[0], float_to_ordered(mn));
            atomicMax(&a.workspace[1], float_to_ordered(mx));
        }
    }
}

// Fixed-stride marcher (BASELINE configs 1/2): the ray's first sample start, t0 = max(t_enter, near) (near if the box is missed)
__device__ __forceinline__ float march_fixed_t0(const float *origins, const float *directions, const float *aabb,
                                                const int64_t r, const float near_plane) {
    const float o[3] = {origins[3 * r], origins[3 * r + 1], origins[3 * r + 2]};
    const float d[3] = {directions[3 * r], directions[3 * r + 1], directions[3 * r + 2]};
    float tmin, tmax;
    const bool hit = ray_aabb(o, d, aabb, tmin, tmax);
    return hit ? fmaxf(tmin, near_plane) : near_plane;
}

// One ray of the fixed-stride marcher by one warp: t advances by repeated float32 addition (bit-exact to the oracle's
// `t = t + step`), every lane runs the same chain and keeps element `lane` of each group of 32, so the stores are
// coalesced (the first version -- one thread per ray, three strided stores per step -- took 58 us for 4096 rays).
__device__ __forceinline__ void march_fixed_warp(const float t0, const int64_t r, const int n_per_ray, const float step,
                                                 float *t_starts, float *t_ends, int32_t *ray_indices, const int lane) {
    const int64_t base = r * n_per_ray;
    float t = t0;
    for (int k0 = 0; k0 < n_per_ray; k0 += 32) {
        float my_s = 0.f, my_e = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float tn = __fadd_rn(t, step);
            if (lane == j) { my_s = t; my_e = tn; }
            t = tn;
        }
        const int k = k0 + lane;
        if (k < n_per_ray) {
            t_starts[base + k] = my_s;
            t_ends[base + k] = my_e;
            ray_indices[base + k] = (int32_t)r;
        }
    }
}

}  // namespace nsb
