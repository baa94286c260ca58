// Jacobian and inverse of the SE(3) deformation field, sm_90a (an extension; DESIGN 4.2e).
//   nsb_deform_jacobian: per point the normalised offset(p_n) = R(p_n) p_n + V v - p_n (deformation_field.py:148-166) and
//                        J = d offset / d p_n, the J whose transpose nsb_deform_input_grad applies.
//   nsb_deform_inverse:  per point the p_n that solves F(p_n) = p_n + D^-1 offset(p_n) - c_n = 0 (D = diag(box extent)),
//                        i.e. the observed position whose warped hash input is the given canonical position c, by damped
//                        Newton inside the kernel.
//
// Forward mode.  A tile of 32 points is a 128-row GEMM: warp w owns points 4w..4w+3, and row 4k + c of the warp is point k's
// primal row (c = 0) or its tangent with respect to p_n[c - 1] (c = 1..3).  Every row goes through the stem with the
// forward slabs of deform_packed_tb (the warp-code columns drop out: the codes do not depend on p):
//   * primal rows exactly as the mma.sync tensor role of the field kernels forms them (posenc with opts.pe_window, fp16
//     activations, code bias of layers 0 / 4 from deform_code_bias[t] or sample_code_bias);
//   * tangent rows start from tangent_scale * d posenc / d p_n (windowed), get no bias, and pass where their primal row's
//     fp16 post-ReLU value is positive; the heads' tangents are divided by tangent_scale;
//   * the SE(3) exponential map and its forward derivative in fp32 on one lane per point, with the conventions of the
//     input-gradient kernel: theta^2 clamped at 1e-4 passes nothing through theta, a NaN warp (the identity in the forward)
//     gets J = 0.
// The weights arrive through one cp.async.bulk / mbarrier ring in order of use: 94 slabs = 24 chunks per evaluation (the
// last one holds the two head slabs).  The chunk sequence is the same for every evaluation, so the ring runs ahead across
// evaluations and tiles; at the end the producer waits for the chunks it issued ahead.
// Newton (nsb_deform_inverse): each evaluation gives F and J at every point's trial position; a trial with a smaller
// |F|inf than the best so far becomes the best and the next trial is best - (I + D^-1 J)^-1 F (3 x 3 solve in fp32, a
// near-singular determinant stops the point), any other trial is replaced by its midpoint with the best.  A tile repeats
// evaluations until all of its points have converged or stopped; finished points ride along unchanged, so the GEMMs never
// diverge.  No atomics, no state across tiles: the result is the same bits on every run.
// The ring GEMM and the SE(3) row function repeat what nsb_deform_vjp.cu has instead of sharing a header with it: moving
// code of that kernel changes its register allocation (DESIGN 4.2c), and its results and spill report are pinned.
#include <algorithm>
#include <cmath>

#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kSlab = 2048, kChunkSlabs = 4, kChunkBytes = kSlab * kChunkSlabs, kStages = 4;
// ring order: the slabs of deform_packed_tb (layers 0 and 4 without their warp-code columns)
constexpr int kF_L0 = 0, kF_L1 = 6, kF_L2 = 22, kF_L3 = 38, kF_L4 = 54, kF_L5 = 76, kF_HEADS = 92, kFSlabs = 94;
constexpr int kChunksPerEval = (kFSlabs + kChunkSlabs - 1) / kChunkSlabs;     // 24, the last one half full
constexpr int kHeadsChunk = kF_HEADS / kChunkSlabs;                         // 23
static_assert(kF_HEADS % kChunkSlabs == 0 && kFSlabs - kF_HEADS == 2 && kHeadsChunk == kChunksPerEval - 1,
              "the head slabs are the last, half-full chunk");
constexpr int kInvThreads = 256;
constexpr int kPointsPerWarp = 4, kPointsPerTile = 8 * kPointsPerWarp;      // 32
constexpr float kTwoPi = 6.283185307179586f;
constexpr float kSingularDet = 1e-6f;

struct InvKArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    float aabb_size[3];
    float tangent_scale;
    // Jacobian mode
    float *offsets, *jacobian;
    // inverse mode
    const float *init;
    int32_t max_iter;
    float tol;
    float *positions, *residual;
    int32_t *iterations, *status;
};

struct alignas(16) WarpScratch {
    float pos[kPointsPerWarp][4];  // normalised trial position xyz, w = row of the code bias (int bits)
    uint4 enc[3][32];              // posenc A fragments [k-tile][lane]
    uint4 act[2][8][32];           // [ping-pong][k-tile][lane]
};

struct alignas(128) SmemInv {
    uint8_t ring[kStages][kChunkBytes];
    uint64_t full[kStages], empty[kStages];
    float bias[6 * 128 + 8];
    WarpScratch ws[8];
};

struct Ring {
    bool producer;         // warp 0, lane 0
    uint32_t gbase;
    const uint8_t *fwd;
    __device__ __forceinline__ void issue(SmemInv &sm, uint32_t gt) const {
        if (producer) {
            const uint32_t s = gt % kStages, kf = gt / kStages, c = gt % kChunksPerEval;
            const uint32_t bytes = c == kHeadsChunk ? kChunkBytes / 2 : kChunkBytes;
            mbar_wait<20>(&sm.empty[s], (kf & 1) ^ 1);      // every warp released the previous use
            mbar_expect_tx(&sm.full[s], bytes);
            bulk_g2s(sm.ring[s], fwd + (size_t)c * kChunkBytes, bytes, &sm.full[s]);
        }
    }
};

// acc[8][4] += A(16 x 16*KT) . ring slabs j0..j0+KT-1 (64 output columns); slabs are consumed strictly in ring order
template <int KT, class AFn>
__device__ __forceinline__ void ring_gemm(float (&acc)[8][4], const int j0, AFn &&afn, SmemInv &sm, const Ring &rf, int lane) {
#pragma unroll 2
    for (int kt = 0; kt < KT; ++kt) {
        const int j = j0 + kt;
        const uint32_t G = rf.gbase + (j >> 2);
        const int stage = G & 3;
        if ((j & 3) == 0) {
            rf.issue(sm, G + (kStages - 1));
            __syncwarp();
            mbar_wait<20>(&sm.full[stage], (G >> 2) & 1);
        }
        uint32_t a[4];
        afn(kt, a);
        const uint4 *slab = reinterpret_cast<const uint4 *>(&sm.ring[stage][(j & 3) * kSlab]);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const uint4 b = slab[p * 32 + lane];
            mma16816(acc[2 * p], a, b.x, b.y);
            mma16816(acc[2 * p + 1], a, b.z, b.w);
        }
        if ((j & 3) == 3) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty[stage]);
        }
    }
}

__device__ __forceinline__ void zero8(float (&acc)[8][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;
}

// One N-half of a stem layer's epilogue into the activation buffer.  Primal rows: bias + ReLU + fp16 (the field kernels'
// relu_store2; CODE: layers 0 / 4 take the per-row code bias from global memory).  Tangent rows: no bias, the element
// passes where the primal row's fp16 output is positive.  The primal row of this lane's rows sits on lane & ~12.
template <int HALF, bool CODE>
__device__ __forceinline__ void relu_tangent_store(const float (&acc)[8][4], uint4 (*dst)[32], const float *sbias,
                                                   const float *gbias, const uint32_t (&off)[2], bool tangent, int q,
                                                   int lane) {
#pragma unroll
    for (int kt = 0; kt < 4; ++kt) {
        uint32_t r[4];
        uint32_t mask = 0;
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            const int nt = 2 * kt + o, col = HALF * 64 + nt * 8 + 2 * q;
            float2 b0, b1;
            if (CODE) {
                b0 = __ldg(reinterpret_cast<const float2 *>(gbias + off[0] + col));
                b1 = __ldg(reinterpret_cast<const float2 *>(gbias + off[1] + col));
            } else {
                b0 = *reinterpret_cast<const float2 *>(sbias + col);
                b1 = b0;
            }
            r[o * 2 + 0] = pack_h2(fmaxf(acc[nt][0] + b0.x, 0.f), fmaxf(acc[nt][1] + b0.y, 0.f));
            r[o * 2 + 1] = pack_h2(fmaxf(acc[nt][2] + b1.x, 0.f), fmaxf(acc[nt][3] + b1.y, 0.f));
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                mask |= ((r[o * 2 + e] & 0x7fffu) != 0u ? 1u : 0u) << (4 * o + 2 * e);
                mask |= ((r[o * 2 + e] & 0x7fff0000u) != 0u ? 1u : 0u) << (4 * o + 2 * e + 1);
            }
        }
        mask = __shfl_sync(0xffffffffu, mask, lane & ~12);
        if (tangent) {
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const int nt = 2 * kt + o;
                const uint32_t mb = mask >> (4 * o);
                r[o * 2 + 0] = pack_h2(mb & 1u ? acc[nt][0] : 0.f, mb & 2u ? acc[nt][1] : 0.f);
                r[o * 2 + 1] = pack_h2(mb & 4u ? acc[nt][2] : 0.f, mb & 8u ? acc[nt][3] : 0.f);
            }
        }
        dst[HALF * 4 + kt][lane] = make_uint4(r[0], r[1], r[2], r[3]);
    }
}

__device__ __forceinline__ void cross(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// pw = R(r) p + V(r) v (util/pytorch3d.py:107-191 + deformation_field.py:95-107) with the field kernels' expressions:
// off = pw - p, a NaN component of pw replaced by p.  Forward derivative for the tangents (dr[k], dv[k]) of p_n[k]:
// jac[i][k] = d off_i / d p_n[k], including the direct term (R - I) e_k.  theta^2 clamped at 1e-4 passes nothing through
// theta; a NaN warp gets jac = 0.
__device__ __forceinline__ void se3_forward_jvp(const float p[3], const float r[3], const float v[3],
                                                const float (&dr)[3][3], const float (&dv)[3][3], float off[3],
                                                float (&jac)[3][3]) {
    const float n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    const bool clamped = !(n2 > 1e-4f);
    const float th = sqrtf(fmaxf(n2, 1e-4f));
    float s, c;
    sincosf(th, &s, &c);
    const float th2 = th * th;
    const float f1 = s / th, f2 = (1.0f - c) / th2, f3 = (th - s) / (th2 * th);
    const float df1 = (th * c - s) / th2;
    const float df2 = (th * s - 2.0f * (1.0f - c)) / (th2 * th);
    const float df3 = ((1.0f - c) * th - 3.0f * (th - s)) / (th2 * th2);
    float A[3], Bv[3], Cv[3], Dv[3];
    cross(r, p, A); cross(r, A, Bv); cross(r, v, Cv); cross(r, Cv, Dv);
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float o = (p[i] + f1 * A[i] + f2 * Bv[i]) + (v[i] + f2 * Cv[i] + f3 * Dv[i]);
        bad = bad || isnan(o);
        off[i] = (isnan(o) ? p[i] : o) - p[i];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float e[3] = {k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f};
        float t0[3], t1[3], dA[3], dB[3], dC[3], dD[3];
        cross(dr[k], p, t0); cross(r, e, t1);
#pragma unroll
        for (int i = 0; i < 3; ++i) dA[i] = t0[i] + t1[i];
        cross(dr[k], A, t0); cross(r, dA, t1);
#pragma unroll
        for (int i = 0; i < 3; ++i) dB[i] = t0[i] + t1[i];
        cross(dr[k], v, t0); cross(r, dv[k], t1);
#pragma unroll
        for (int i = 0; i < 3; ++i) dC[i] = t0[i] + t1[i];
        cross(dr[k], Cv, t0); cross(r, dC, t1);
#pragma unroll
        for (int i = 0; i < 3; ++i) dD[i] = t0[i] + t1[i];
        const float dth = clamped ? 0.f : (r[0] * dr[k][0] + r[1] * dr[k][1] + r[2] * dr[k][2]) / th;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float j = dth * (df1 * A[i] + df2 * (Bv[i] + Cv[i]) + df3 * Dv[i]) + f1 * dA[i] + f2 * (dB[i] + dC[i]) +
                            f3 * dD[i] + dv[k][i];
            jac[i][k] = bad ? 0.f : j;
        }
    }
}

template <bool INVERSE>
__global__ void __launch_bounds__(kInvThreads, 1) deform_inv_kernel(const __grid_constant__ InvKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemInv &sm = *reinterpret_cast<SmemInv *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int64_t n = K.S.n_samples_dev ? min(*K.S.n_samples_dev, K.S.n_samples) : K.S.n_samples;
    const int64_t n_tiles = (n + kPointsPerTile - 1) / kPointsPerTile;
    const int64_t my_tiles = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    for (int i = tid; i < 6 * 128 + 8; i += kInvThreads) sm.bias[i] = K.P.deform_bias[i];
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], 8); }
        mbar_fence_init();
    }
    __syncthreads();
    if (my_tiles == 0) return;
    Ring rf;
    rf.producer = tid == 0;
    rf.fwd = reinterpret_cast<const uint8_t *>(K.P.deform_packed_tb);
    rf.gbase = 0;
    for (uint32_t c = 0; c < kStages - 1; ++c) rf.issue(sm, c);
    __syncwarp();
    WarpScratch &ws = sm.ws[warp];
    const float amin[3] = {K.P.aabb[0], K.P.aabb[1], K.P.aabb[2]};
    const float *const gcb = K.S.sample_code_bias ? K.S.sample_code_bias : K.P.deform_code_bias;
    const float ts = K.tangent_scale, inv_ts = 1.0f / K.tangent_scale;
    // rows g / g+8 of this lane: points (g >> 2) and (g >> 2) + 2 of the warp, component c = g & 3 (0: primal)
    const int comp = g & 3;
    const bool tangent = comp != 0;
    // the lane that runs the SE(3) map of point `pt` holds its primal row: lanes 0, 16, 1, 17 for points 0..3
    const bool se3_lane = (lane & 14) == 0;
    const int pt = ((lane >> 4) & 1) | ((lane & 1) << 1);
    uint32_t evals = 0;

#pragma unroll 1
    for (int64_t it = 0; it < my_tiles; ++it) {
        const int64_t tile = blockIdx.x + it * gridDim.x;
        const int64_t s = tile * kPointsPerTile + warp * kPointsPerWarp + pt;     // this SE(3) lane's point
        const bool live = se3_lane && s < n;
        // per-point state on the SE(3) lane (world positions, so that an untouched point keeps its bits)
        float trial[3] = {0.f, 0.f, 0.f}, best[3] = {0.f, 0.f, 0.f}, cn[3] = {0.f, 0.f, 0.f};
        float rbest = INFINITY;
        int32_t iters = 0, stat = live ? -1 : 1;    // -1: running; 0 converged, 1 not converged, 2 singular
        int tsi = 0;
        if (se3_lane) {
            float tt = 0.f;
            if (live) {
#pragma unroll
                for (int k = 0; k < 3; ++k) trial[k] = K.S.positions[3 * s + k];
                if (K.S.sample_times) tt = K.S.sample_times[s];
            }
            tsi = sample_timestep(tt, K.P.n_timesteps);
            if (K.S.sample_code_bias) tsi = (int)min(s, n - 1);     // per-sample warp codes: the bias rows are per sample
            if (INVERSE && live) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    cn[k] = box_coord(trial[k], amin[k], K.aabb_size[k]);
                    if (K.init) trial[k] = K.init[3 * s + k];
                    best[k] = trial[k];
                }
            }
        }
#pragma unroll 1
        for (;;) {
            rf.gbase = evals * kChunksPerEval;
            ++evals;
            __syncwarp();
            if (se3_lane) {
#pragma unroll
                for (int k = 0; k < 3; ++k) ws.pos[pt][k] = box_coord(trial[k], amin[k], K.aabb_size[k]);
                ws.pos[pt][3] = __int_as_float(tsi);
            }
            __syncwarp();
            float pn[2][3];    // the points of rows g / g+8
            uint32_t cb[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int ph = (g >> 2) + 2 * h;
                pn[h][0] = ws.pos[ph][0]; pn[h][1] = ws.pos[ph][1]; pn[h][2] = ws.pos[ph][2];
                cb[h] = (uint32_t)__float_as_int(ws.pos[ph][3]) * 256u;
            }
            // ---- windowed posenc fragments: primal rows as the field kernels form them, tangent rows d/dp_n[comp-1] ----
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) {
                uint32_t w4[4];
#pragma unroll
                for (int hi = 0; hi < 2; ++hi) {
                    const int i = kt * 8 + hi * 4 + q;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float e0 = 0.f, e1 = 0.f;
                        if (i < 21) {
                            const int d = i / 7, j = i - d * 7;
                            const float pd = d == 0 ? pn[h][0] : (d == 1 ? pn[h][1] : pn[h][2]);
                            const float arg = (kTwoPi * pd) * (float)(1 << j);
                            const float wj = K.O.pe_window[j];
                            if (!tangent) {
                                e0 = wj * sinf(arg);
                                e1 = wj * sinf(arg + 1.5707963267948966f);
                            } else if (d == comp - 1) {
                                float sn, cs;
                                sincosf(arg, &sn, &cs);
                                const float f = (ts * wj) * (kTwoPi * (float)(1 << j));
                                e0 = f * cs;
                                e1 = -f * sn;
                            }
                        } else if (i == 21) {
                            e0 = !tangent ? kTwoPi * pn[h][0] : (comp == 1 ? ts * kTwoPi : 0.f);
                            e1 = !tangent ? kTwoPi * pn[h][1] : (comp == 2 ? ts * kTwoPi : 0.f);
                        } else if (i == 22) {
                            e0 = !tangent ? kTwoPi * pn[h][2] : (comp == 3 ? ts * kTwoPi : 0.f);
                        }
                        w4[hi * 2 + h] = pack_h2(e0, e1);
                    }
                }
                ws.enc[kt][lane] = make_uint4(w4[0], w4[1], w4[2], w4[3]);
            }
            auto in_a = [&](int kt, uint32_t(&a)[4]) {
                const uint4 v = ws.enc[kt][lane];
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
            };
            auto buf0 = [&](int kt, uint32_t(&a)[4]) {
                const uint4 v = ws.act[0][kt][lane];
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
            };
            auto buf1 = [&](int kt, uint32_t(&a)[4]) {
                const uint4 v = ws.act[1][kt][lane];
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
            };
            auto skip_a = [&](int kt, uint32_t(&a)[4]) {
                if (kt < 8) buf1(kt, a); else in_a(kt - 8, a);
            };
            // ---- six stem layers, primal and tangent rows together ----
            float acc[8][4];
            zero8(acc); ring_gemm<3>(acc, kF_L0, in_a, sm, rf, lane); relu_tangent_store<0, true>(acc, ws.act[0], nullptr, gcb, cb, tangent, q, lane);
            zero8(acc); ring_gemm<3>(acc, kF_L0 + 3, in_a, sm, rf, lane); relu_tangent_store<1, true>(acc, ws.act[0], nullptr, gcb, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L1, buf0, sm, rf, lane); relu_tangent_store<0, false>(acc, ws.act[1], sm.bias + 1 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L1 + 8, buf0, sm, rf, lane); relu_tangent_store<1, false>(acc, ws.act[1], sm.bias + 1 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L2, buf1, sm, rf, lane); relu_tangent_store<0, false>(acc, ws.act[0], sm.bias + 2 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L2 + 8, buf1, sm, rf, lane); relu_tangent_store<1, false>(acc, ws.act[0], sm.bias + 2 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L3, buf0, sm, rf, lane); relu_tangent_store<0, false>(acc, ws.act[1], sm.bias + 3 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L3 + 8, buf0, sm, rf, lane); relu_tangent_store<1, false>(acc, ws.act[1], sm.bias + 3 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<11>(acc, kF_L4, skip_a, sm, rf, lane); relu_tangent_store<0, true>(acc, ws.act[0], nullptr, gcb + 128, cb, tangent, q, lane);
            zero8(acc); ring_gemm<11>(acc, kF_L4 + 11, skip_a, sm, rf, lane); relu_tangent_store<1, true>(acc, ws.act[0], nullptr, gcb + 128, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L5, buf0, sm, rf, lane); relu_tangent_store<0, false>(acc, ws.act[1], sm.bias + 5 * 128, nullptr, cb, tangent, q, lane);
            zero8(acc); ring_gemm<8>(acc, kF_L5 + 8, buf0, sm, rf, lane); relu_tangent_store<1, false>(acc, ws.act[1], sm.bias + 5 * 128, nullptr, cb, tangent, q, lane);
            // ---- heads: (v, r) of rows g / g+8 from the last, half-full chunk of the evaluation ----
            float hacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            {
                const uint32_t G = rf.gbase + kHeadsChunk;
                const int stage = G & 3;
                rf.issue(sm, G + (kStages - 1));
                __syncwarp();
                mbar_wait<20>(&sm.full[stage], (G >> 2) & 1);
                const uint4 *hw = reinterpret_cast<const uint4 *>(&sm.ring[stage][0]);
#pragma unroll
                for (int kt = 0; kt < 8; ++kt) {
                    const uint4 bw = hw[kt * 32 + lane];
                    uint32_t a[4];
                    buf1(kt, a);
                    mma16816(hacc[0], a, bw.x, bw.y);
                    mma16816(hacc[1], a, bw.z, bw.w);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&sm.empty[stage]);
            }
            const float hb0 = tangent ? 0.f : sm.bias[6 * 128 + 2 * q], hb1 = tangent ? 0.f : sm.bias[6 * 128 + 2 * q + 1];
            const float hs = tangent ? inv_ts : 1.0f;
            const float c0 = (hacc[0][0] + hb0) * hs, c1 = (hacc[0][1] + hb1) * hs;
            const float c2 = (hacc[0][2] + hb0) * hs, c3 = (hacc[0][3] + hb1) * hs;
            const int rsel = q & 1;
            float vr[6];       // lanes q = 0 / 1: (v, r) of row g / g+8
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int srcl = (lane & ~3) | k;
                const float a0 = __shfl_sync(0xffffffffu, c0, srcl), a1 = __shfl_sync(0xffffffffu, c1, srcl);
                const float b0 = __shfl_sync(0xffffffffu, c2, srcl), b1 = __shfl_sync(0xffffffffu, c3, srcl);
                vr[2 * k] = rsel ? b0 : a0;
                vr[2 * k + 1] = rsel ? b1 : a1;
            }
            // the tangent rows of point pt sit 4, 8, 12 lanes above its primal row
            float dv[3][3], dr[3][3];
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    dv[c][k] = __shfl_down_sync(0xffffffffu, vr[k], 4 * (c + 1));
                    dr[c][k] = __shfl_down_sync(0xffffffffu, vr[3 + k], 4 * (c + 1));
                }
            bool running = false;
            if (se3_lane) {
                const float p[3] = {ws.pos[pt][0], ws.pos[pt][1], ws.pos[pt][2]};
                const float v[3] = {vr[0], vr[1], vr[2]}, r[3] = {vr[3], vr[4], vr[5]};
                float off[3], jac[3][3];
                se3_forward_jvp(p, r, v, dr, dv, off, jac);
                if (!INVERSE) {
                    if (live) {
#pragma unroll
                        for (int i = 0; i < 3; ++i) {
                            K.offsets[3 * s + i] = off[i];
#pragma unroll
                            for (int k = 0; k < 3; ++k) K.jacobian[9 * s + 3 * i + k] = jac[i][k];
                        }
                    }
                } else if (stat < 0) {
                    // F = the warped hash input (world position + normalised offset, as the field kernels form it) - c_n
                    float F[3];
                    bool bad = false;
                    float res = 0.f;
#pragma unroll
                    for (int i = 0; i < 3; ++i) {
                        F[i] = box_coord(__fadd_rn(trial[i], off[i]), amin[i], K.aabb_size[i]) - cn[i];
                        bad = bad || isnan(F[i]);
                        res = fmaxf(res, fabsf(F[i]));
                    }
                    if (bad) res = INFINITY;
                    const bool better = res < rbest;
                    if (better) {
                        rbest = res;
#pragma unroll
                        for (int k = 0; k < 3; ++k) best[k] = trial[k];
                    }
                    if (rbest < K.tol) {
                        stat = 0;
                    } else if (iters >= K.max_iter) {
                        stat = 1;
                    } else if (better) {
                        // Newton from the best: (I + D^-1 J) delta = F, in normalised units
                        float M[3][3];
#pragma unroll
                        for (int i = 0; i < 3; ++i)
#pragma unroll
                            for (int k = 0; k < 3; ++k) M[i][k] = (i == k ? 1.f : 0.f) + jac[i][k] / K.aabb_size[i];
                        const float a00 = M[1][1] * M[2][2] - M[1][2] * M[2][1];
                        const float a01 = M[0][2] * M[2][1] - M[0][1] * M[2][2];
                        const float a02 = M[0][1] * M[1][2] - M[0][2] * M[1][1];
                        const float a10 = M[1][2] * M[2][0] - M[1][0] * M[2][2];
                        const float a11 = M[0][0] * M[2][2] - M[0][2] * M[2][0];
                        const float a12 = M[0][2] * M[1][0] - M[0][0] * M[1][2];
                        const float a20 = M[1][0] * M[2][1] - M[1][1] * M[2][0];
                        const float a21 = M[0][1] * M[2][0] - M[0][0] * M[2][1];
                        const float a22 = M[0][0] * M[1][1] - M[0][1] * M[1][0];
                        const float det = M[0][0] * a00 + M[0][1] * a10 + M[0][2] * a20;
                        if (!(fabsf(det) > kSingularDet)) {
                            stat = 2;
                        } else {
                            const float id = 1.0f / det;
                            const float d0 = (a00 * F[0] + a01 * F[1] + a02 * F[2]) * id;
                            const float d1 = (a10 * F[0] + a11 * F[1] + a12 * F[2]) * id;
                            const float d2 = (a20 * F[0] + a21 * F[1] + a22 * F[2]) * id;
                            trial[0] = best[0] - d0 * K.aabb_size[0];
                            trial[1] = best[1] - d1 * K.aabb_size[1];
                            trial[2] = best[2] - d2 * K.aabb_size[2];
                            ++iters;
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < 3; ++k) trial[k] = 0.5f * (best[k] + trial[k]);
                        ++iters;
                    }
                    running = stat < 0;
                }
            }
            if (!INVERSE || !__syncthreads_or(running)) break;
        }
        if (INVERSE && live) {
#pragma unroll
            for (int k = 0; k < 3; ++k) K.positions[3 * s + k] = best[k];
            K.residual[s] = rbest;
            K.iterations[s] = iters;
            K.status[s] = stat;
        }
    }
    // the ring ran ahead by kStages - 1 chunks: wait for them before the CTA's shared memory goes away
    if (rf.producer) {
        const uint32_t consumed = evals * kChunksPerEval;
        for (uint32_t gt = consumed; gt < consumed + kStages - 1; ++gt) mbar_wait<20>(&sm.full[gt % kStages], (gt / kStages) & 1);
    }
}

template <bool INVERSE>
int launch(const char *who, const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
           const InvKArgs &K0, cudaStream_t st) {
    InvKArgs K = K0;
    K.P = *params; K.O = *opts; K.S = *samples;
    for (int k = 0; k < 3; ++k) K.aabb_size[k] = params->aabb[3 + k] - params->aabb[k];
    const int smem = (int)sizeof(SmemInv);
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(deform_inv_kernel<INVERSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) { set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e)); return 1; }
        configured = true;
    }
    const int64_t n_tiles = (samples->n_samples + kPointsPerTile - 1) / kPointsPerTile;
    const int n_ctas = (int)std::min<int64_t>(n_tiles, num_sms());
    deform_inv_kernel<INVERSE><<<n_ctas, kInvThreads, smem, st>>>(K);
    return check_launch(INVERSE ? "deform_inv_kernel<inverse>" : "deform_inv_kernel<jacobian>");
}

// Checks common to both entry points; returns 1 with the error set.
int check_common(const char *who, const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                 float tangent_scale) {
    if (!params || !opts || !samples) { set_error("%s: null argument", who); return 1; }
    if (check_field_params(who, params) || check_samples(who, samples)) return 1;
    if (samples->origins || !samples->positions) {
        set_error("%s: positions-based samples only", who);
        return 1;
    }
    if (!params->deform_packed_tb || !params->deform_bias || (!params->deform_code_bias && !samples->sample_code_bias)) {
        set_error("%s: missing deformation parameters", who);
        return 1;
    }
    if (!(tangent_scale > 0.f) || !std::isfinite(tangent_scale)) {
        set_error("%s: tangent_scale must be finite and > 0", who);
        return 1;
    }
    if (samples->sample_code_bias && samples->n_samples > ((int64_t)1 << 24)) {
        set_error("%s: per-sample code bias: at most 2^24 samples", who);
        return 1;
    }
    return 0;
}

}  // namespace
}  // namespace nsb

using namespace nsb;

extern "C" int nsb_deform_jacobian(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                   const nsb_deform_jac_args *args, void *stream) {
    const char *who = "nsb_deform_jacobian";
    if (!args) { set_error("%s: null argument", who); return 1; }
    if (check_common(who, params, opts, samples, args->tangent_scale)) return 1;
    if (!args->offsets || !args->jacobian) { set_error("%s: null output", who); return 1; }
    if (samples->n_samples <= 0) return 0;
    InvKArgs K = {};
    K.tangent_scale = args->tangent_scale;
    K.offsets = args->offsets;
    K.jacobian = args->jacobian;
    return launch<false>(who, params, opts, samples, K, (cudaStream_t)stream);
}

extern "C" int nsb_deform_inverse(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                  const nsb_deform_inv_args *args, void *stream) {
    const char *who = "nsb_deform_inverse";
    if (!args) { set_error("%s: null argument", who); return 1; }
    if (check_common(who, params, opts, samples, args->tangent_scale)) return 1;
    if (args->max_iter < 1 || args->max_iter > 64) {
        set_error("%s: max_iter must be in 1..64, got %d", who, (int)args->max_iter);
        return 1;
    }
    if (!(args->tol > 0.f) || !std::isfinite(args->tol)) { set_error("%s: tol must be finite and > 0", who); return 1; }
    if (!args->positions || !args->residual || !args->iterations || !args->status) {
        set_error("%s: null output", who);
        return 1;
    }
    if (samples->n_samples <= 0) return 0;
    InvKArgs K = {};
    K.tangent_scale = args->tangent_scale;
    K.init = args->init;
    K.max_iter = args->max_iter;
    K.tol = args->tol;
    K.positions = args->positions;
    K.residual = args->residual;
    K.iterations = args->iterations;
    K.status = args->status;
    return launch<true>(who, params, opts, samples, K, (cudaStream_t)stream);
}
