// Shared device helpers for libnsb (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "nsb.h"

namespace nsb {

void set_error(const char *fmt, ...);
int check_launch(const char *what);
// multiprocessors of the current device, queried once
int num_sms();
// Host checks shared by the entry points; each returns 1 with the error set (prefixed by `who`) or 0.
// check_field_params: 16 levels, n_timesteps >= 1, and timestep * frame_stride + entry fits the gather's 32 bits.
// check_samples: a sample source, and ray-based samples with all of directions, t_starts, t_ends, ray_indices.
int check_field_params(const char *who, const nsb_field_params *p);
int check_samples(const char *who, const nsb_samples *s);
// nsb_deform_vjp.cu: d_pn = J^T (u_scale * u) of the deformation (nsb_deform_input_grad) after the entry point's own
// checks; errors are prefixed by `who`.
int launch_deform_input_grad(const char *who, const nsb_field_params *params, const nsb_field_opts *opts,
                             const nsb_samples *samples, const nsb_deform_vjp_args *args, const float u_scale[3],
                             cudaStream_t st);
// nsb_render.cu: the occupancy march as ONE cooperative launch (count | scan | fill); leaves packed_info, the packed
// samples (below `capacity`) and, in the workspace header, n_total / status.  Zeroes and uses hdr->barrier.
int launch_march_occ_coop(const nsb_march_args &M, int64_t *packed_info, nsb_render_ws_header *hdr, int64_t *partials,
                          int64_t capacity, float *scratch, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// Hash-grid addressing (tcnn grid.h) and the sample inputs, shared by the kernels: the backward, the normals pass and the
// stand-alone blend are only right if they pick the forward gather's corners and weights bit for bit.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kPrimeY = 2654435761u;
constexpr uint32_t kPrimeZ = 805459861u;

// Index of corner (cx, cy, cz) within a level: (x ^ y*kPrimeY ^ z*kPrimeZ) mod 2^log2T on hashed levels (their entries
// are 2^log2T, checked on the host), else x + y*res + z*res^2 mod entries, which is < 2*entries for corner coords <= res,
// so one conditional subtract.
__device__ __forceinline__ uint32_t grid_index(bool hashed, uint32_t res, uint32_t entries, uint32_t cx, uint32_t cy,
                                               uint32_t cz) {
    const uint32_t ih = (cx ^ (cy * kPrimeY) ^ (cz * kPrimeZ)) & (entries - 1);
    uint32_t id = cx + cy * res + cz * res * res;
    id = id >= entries ? id - entries : id;
    return hashed ? ih : id;
}

// The timestep of a sample time t in [0, 1]: round(t * (T - 1)), clamped to [0, T - 1].
__device__ __forceinline__ int sample_timestep(float t, int n_timesteps) {
    const int ts = __float2int_rn(__fmul_rn(t, (float)(n_timesteps - 1)));
    return min(max(ts, 0), n_timesteps - 1);
}

// Continuous time (DESIGN 4.2g, the linear render kernels): the fractional timestep u = clamp(t * (T - 1), 0, T - 1),
// snapped to the nearest integer within NSB_TIME_SNAP timesteps (fp32 times k / (T - 1) land a few ulp off k).  A
// snapped u equals sample_timestep(t).  The rows interpolated are floor(u) and min(floor(u) + 1, T - 1) at
// lam = u - floor(u) (exact in fp32); ops.time_lerp is the host mirror.
#define NSB_TIME_SNAP 0.0009765625f     // 2^-10 timesteps
__device__ __forceinline__ float sample_time_u(float t, int n_timesteps) {
    const float tm = (float)(n_timesteps - 1);
    const float u = fminf(fmaxf(__fmul_rn(t, tm), 0.f), tm);
    const float r = rintf(u);
    return fabsf(u - r) <= NSB_TIME_SNAP ? r : u;
}
// (1 - lam) a + lam b, exactly a at lam = 0
__device__ __forceinline__ float time_lerp(float a, float b, float lam) { return fmaf(lam, b - a, a); }

// One axis of a ray sample's position: o + d * (t_start + t_end) / 2, with mid = t_start + t_end (no FMA, like the oracle).
__device__ __forceinline__ float ray_midpoint(float o, float d, float mid) {
    return __fadd_rn(o, __fmul_rn(__fmul_rn(d, mid), 0.5f));
}

// One axis of a world position in box coordinates: (p - aabb_min) / extent.
__device__ __forceinline__ float box_coord(float p, float aabb_min, float extent) {
    return __fdiv_rn(__fsub_rn(p, aabb_min), extent);
}

// ---------------------------------------------------------------------------------------------
// mbarrier / bulk-copy (TMA 1-D) primitives
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
// Spin with back-off: a waiting warp must not burn issue slots the gather warps need
// (an idle producer spinning without sleep takes a large share of the issued instructions).
#ifndef NSB_SPIN_LIMIT
#define NSB_SPIN_LIMIT (1u << 27)   // ~several seconds: a protocol bug traps instead of hanging the GPU
#endif
template <int SLEEP_NS>
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
#ifdef NSB_NO_SPIN_GUARD
    // The forward kernel opts out: the counter costs a live register at every wait site, and with it spills.  The
    // backward kernels keep the guard.
    while (!mbar_try_wait(bar, parity)) {
        if (SLEEP_NS > 0) __nanosleep(SLEEP_NS);
    }
#else
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (SLEEP_NS > 0) __nanosleep(SLEEP_NS);
        if (++spins > NSB_SPIN_LIMIT) __trap();
    }
#endif
}
// global -> shared bulk async copy (UBLKCP), completion signalled on an mbarrier
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---------------------------------------------------------------------------------------------
// tensor-core MMA m16n8k16 (fp16 x fp16 -> fp32).  Fragment layouts (g = lane>>2, q = lane&3):
//   A: a0=(row g, k 2q..2q+1) a1=(row g+8, same k) a2=(row g, k 2q+8..) a3=(row g+8, k 2q+8..)
//   B: b0=(k 2q..2q+1, n g)   b1=(k 2q+8.., n g)
//   C: c0=(row g, col 2q) c1=(row g, col 2q+1) c2=(row g+8, col 2q) c3=(row g+8, col 2q+1)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t u) {
    __half2 h = *reinterpret_cast<__half2 *>(&u);
    return __half22float2(h);
}

// ordered-int encoding of floats for atomicMin/Max
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// ---------------------------------------------------------------------------------------------
// ray / aabb slab test in float32 without fused multiply-add (bit-exact to the oracle's numpy)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool ray_aabb(const float o[3], const float d[3], const float *aabb, float &tmin,
                                         float &tmax) {
    tmin = -INFINITY;
    tmax = INFINITY;
    bool any_lo = false, any_hi = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float inv = __fdiv_rn(1.0f, d[k]);
        float t0 = __fmul_rn(__fsub_rn(aabb[k], o[k]), inv);
        float t1 = __fmul_rn(__fsub_rn(aabb[3 + k], o[k]), inv);
        if (isnan(t0) || isnan(t1)) continue;  // 0*inf slab: ignored (oracle: np.minimum -> nanmax)
        float lo = fminf(t0, t1), hi = fmaxf(t0, t1);
        tmin = any_lo ? fmaxf(tmin, lo) : lo; any_lo = true;
        tmax = any_hi ? fminf(tmax, hi) : hi; any_hi = true;
    }
    return tmin <= tmax;
}

}  // namespace nsb
