// Input-position gradient of the SE(3) deformation field, sm_90a: d_pn = J^T u per sample, with
// offset(p_n) = R(p_n) p_n + V v - p_n (deformation_field.py:148-166), J = d offset / d p_n and u a given cotangent.
// J runs through the windowed positional encoding, the six stem layers, both heads and the SE(3) exponential map, plus
// the direct dependence (R - I) p_n.  Used for observation-space surface normals (nsb_normals_forward) and exposed as
// nsb_deform_input_grad.
//
// One CTA = 8 warps = one 128-sample tile, persistent over tiles; warp w owns rows 16w..16w+15 and never talks to the
// other warps except through the weight ring.
//   * forward RECOMPUTED per tile with the operand rounding of the mma.sync tensor role of the field kernels (posenc with
//     opts.pe_window, fp16 activations, code bias of layers 0 / 4 from deform_code_bias[t] or sample_code_bias): the
//     render kernels save no activations, and one mode serves every caller.  Only the ReLU masks (128 bits per row and
//     layer, 12 registers per lane) and (r, v) are kept;
//   * SE(3) exp-map backward in fp32 per row for (d r, d v), and the direct term (R - I)^T u;
//   * the delta chain heads -> L5 -> ... -> L1 on mma.sync m16n8k16 with the TRANSPOSED hidden blocks of pack_deform_bwd,
//     ping-ponging through the warp's activation buffers.  Forward and transposed slabs arrive through one
//     cp.async.bulk / mbarrier ring in order of use (176 slabs = 44 chunks per tile; the code-column blocks of the
//     transposed pack are skipped, nothing here needs a code gradient);
//   * posenc backward: d enc = delta_0 . W0[:, posenc] + delta_4 . W4[:, posenc] against two [128 -> 48] transposed blocks
//     resident in shared memory (pack_deform_pe_t), then the chain rule through sin / cos and the 2 pi x columns.
// No weight gradients, no atomics, no state across tiles: the result is the same bits on every run.
// The SE(3) row function and the ring GEMM repeat what nsb_deform_bwd.cu has instead of sharing a header with it: moving
// code of that kernel changes its register allocation (DESIGN 4.1), and its results and spill report are pinned.
#include <algorithm>

#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kSlab = 2048, kChunkSlabs = 4, kChunkBytes = kSlab * kChunkSlabs, kStages = 4;
// ring order, forward part: the slabs of deform_packed_tb (layers 0 and 4 without their warp-code columns)
constexpr int kF_L0 = 0, kF_L1 = 6, kF_L2 = 22, kF_L3 = 38, kF_L4 = 54, kF_L5 = 76, kF_HEADS = 92, kFSlabs = 94;
// ring order, backward part: transposed heads, L5, L4 hidden, L3, L2, L1 of pack_deform_bwd.  That pack also holds the code
// columns of layer 4 (its slabs 34..49) and of layer 0 (98..113); they are left out.
constexpr int kB_HEADS = kFSlabs, kB_L5 = kB_HEADS + 2, kB_L4H = kB_L5 + 16, kB_L3 = kB_L4H + 16, kB_L2 = kB_L3 + 16,
              kB_L1 = kB_L2 + 16, kSlabsPerTile = kB_L1 + 16;
constexpr int kChunksPerTile = kSlabsPerTile / kChunkSlabs;       // 44
constexpr int kSplitChunk = kFSlabs / kChunkSlabs;                // 23: two forward slabs (the heads), two transposed
constexpr int kTSkipAt = 34, kTSkip = 16;
static_assert(kSlabsPerTile % kChunkSlabs == 0 && kFSlabs % kChunkSlabs == 2 && kF_HEADS % kChunkSlabs == 0 &&
              (kTSkipAt + kFSlabs) % kChunkSlabs == 0, "chunk boundaries of the ring");
constexpr int kPeU4 = 8 * 3 * 32;     // one transposed posenc block: 8 k-tiles x 3 n-tile pairs x 32 lanes
constexpr int kVjpThreads = 256;
constexpr float kTwoPi = 6.283185307179586f;

struct VjpKArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    nsb_deform_vjp_args V;
    float aabb_size[3];
    float u_scale[3];      // per-axis factor on u (1, or 1 / extent when the caller's vectors are unit normals)
};

struct alignas(16) WarpScratch {
    float pos[16][4];      // normalised position xyz, w = row of the code bias (int bits)
    uint4 enc[3][32];      // posenc A fragments [k-tile][lane]
    uint4 act[2][8][32];   // [ping-pong][k-tile][lane]: activations forward, deltas backward (lane-private)
};

struct alignas(128) SmemVjp {
    uint8_t ring[kStages][kChunkBytes];
    uint64_t full[kStages], empty[kStages];
    float bias[6 * 128 + 8];
    uint4 pe_t[2][kPeU4];  // transposed posenc columns of layer 0 | layer 4
    WarpScratch ws[8];
};

struct Ring {
    bool producer;         // warp 0, lane 0
    uint32_t gbase, total;
    const uint8_t *fwd, *bwd;
    __device__ __forceinline__ void issue(SmemVjp &sm, uint32_t gt) const {
        if (producer && gt < total) {
            const uint32_t s = gt % kStages, kf = gt / kStages, c = gt % kChunksPerTile;
            mbar_wait<20>(&sm.empty[s], (kf & 1) ^ 1);      // every warp released the previous use
            mbar_expect_tx(&sm.full[s], kChunkBytes);
            if (c < kSplitChunk) {
                bulk_g2s(sm.ring[s], fwd + (size_t)c * kChunkBytes, kChunkBytes, &sm.full[s]);
            } else if (c == kSplitChunk) {
                bulk_g2s(sm.ring[s], fwd + (size_t)c * kChunkBytes, kChunkBytes / 2, &sm.full[s]);
                bulk_g2s(sm.ring[s] + kChunkBytes / 2, bwd, kChunkBytes / 2, &sm.full[s]);
            } else {
                const uint32_t b = c * kChunkSlabs - kFSlabs;
                bulk_g2s(sm.ring[s], bwd + (size_t)(b < kTSkipAt ? b : b + kTSkip) * kSlab, kChunkBytes, &sm.full[s]);
            }
        }
    }
};

// acc[8][4] += A(16 x 16*KT) . ring slabs j0..j0+KT-1 (64 output columns); slabs are consumed strictly in ring order
template <int KT, class AFn>
__device__ __forceinline__ void ring_gemm(float (&acc)[8][4], const int j0, AFn &&afn, SmemVjp &sm, const Ring &rf, int lane) {
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

// bit e of the result: element e (low / high half of x, y, z, w) of the post-ReLU fp16 fragment is > 0
__device__ __forceinline__ uint32_t pos_bits(const uint4 v) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        m |= ((w[k] & 0x7fffu) != 0u ? 1u : 0u) << (2 * k);
        m |= ((w[k] & 0x7fff0000u) != 0u ? 1u : 0u) << (2 * k + 1);
    }
    return m;
}

// bias + ReLU + pack one N-half into the activation buffer (the field kernels' relu_store2), and the half's ReLU bits:
// byte kt of `mask` = pos_bits of k-tile HALF*4 + kt.  CODE: layers 0 / 4 take the per-row code bias from global memory.
template <int HALF, bool CODE>
__device__ __forceinline__ uint32_t relu_store(const float (&acc)[8][4], uint4 (*dst)[32], const float *sbias,
                                               const float *gbias, const uint32_t (&off)[2], int q, int lane) {
    uint32_t mask = 0;
#pragma unroll
    for (int kt = 0; kt < 4; ++kt) {
        uint32_t r[4];
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
        }
        const uint4 v = make_uint4(r[0], r[1], r[2], r[3]);
        dst[HALF * 4 + kt][lane] = v;
        mask |= pos_bits(v) << (8 * kt);
    }
    return mask;
}

// delta of the layer below: the accumulators of one N-half times the ReLU bits of that layer's output, as A fragments
template <int HALF>
__device__ __forceinline__ void delta_store(const float (&acc)[8][4], uint4 (*dst)[32], uint32_t mask, int lane) {
#pragma unroll
    for (int kt = 0; kt < 4; ++kt) {
        const uint32_t mb = mask >> (8 * kt);
        uint4 v;
        v.x = pack_h2(mb & 1u ? acc[2 * kt][0] : 0.f, mb & 2u ? acc[2 * kt][1] : 0.f);
        v.y = pack_h2(mb & 4u ? acc[2 * kt][2] : 0.f, mb & 8u ? acc[2 * kt][3] : 0.f);
        v.z = pack_h2(mb & 16u ? acc[2 * kt + 1][0] : 0.f, mb & 32u ? acc[2 * kt + 1][1] : 0.f);
        v.w = pack_h2(mb & 64u ? acc[2 * kt + 1][2] : 0.f, mb & 128u ? acc[2 * kt + 1][3] : 0.f);
        dst[HALF * 4 + kt][lane] = v;
    }
}

__device__ __forceinline__ void cross(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// Backward of pw = R(r) p + V(r) v (util/pytorch3d.py:107-191 + deformation_field.py:95-107) for g = dL/dpw: dr, dv and
// dp = (R - I)^T g, the direct dependence of pw - p on p.  theta^2 is clamped at 1e-4 (no gradient through theta
// below it); a NaN warp is replaced by the identity in the forward, so such a row gets no gradient at all.
__device__ __forceinline__ void se3_input_vjp(const float p[3], const float r[3], const float v[3], const float g[3],
                                              float dr[3], float dv[3], float dp[3]) {
    const float n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    const bool clamped = !(n2 > 1e-4f);
    const float th = sqrtf(fmaxf(n2, 1e-4f));
    float s, c;
    sincosf(th, &s, &c);
    const float th2 = th * th;
    const float f1 = s / th, f2 = (1.0f - c) / th2, f3 = (th - s) / (th2 * th);
    float A[3], Bv[3], Cv[3], Dv[3], gxr[3], rxg[3], rrg[3], t0[3], t1[3], t2[3], t3[3], t4[3], t5[3];
    cross(r, p, A); cross(r, A, Bv); cross(r, v, Cv); cross(r, Cv, Dv);
    cross(g, r, gxr); cross(r, g, rxg); cross(r, rxg, rrg);
    cross(p, g, t0);      // d/dr [g.(r x p)]
    cross(A, g, t1);      // d/dr [g.(r x a)], a = r x p fixed
    cross(p, gxr, t2);    //   ... through a
    cross(v, g, t3);      // d/dr [g.(r x v)]
    cross(Cv, g, t4);     // d/dr [g.(r x w)], w = r x v fixed
    cross(v, gxr, t5);    //   ... through w
    float dth = 0.f;
    if (!clamped) {
        const float df1 = (th * c - s) / th2;
        const float df2 = (th * s - 2.0f * (1.0f - c)) / (th2 * th);
        const float df3 = ((1.0f - c) * th - 3.0f * (th - s)) / (th2 * th2);
#pragma unroll
        for (int k = 0; k < 3; ++k) dth += g[k] * (df1 * A[k] + df2 * (Bv[k] + Cv[k]) + df3 * Dv[k]);
    }
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float pw = (p[k] + f1 * A[k] + f2 * Bv[k]) + (v[k] + f2 * Cv[k] + f3 * Dv[k]);
        bad = bad || isnan(pw);
        dv[k] = g[k] + f2 * gxr[k] + f3 * rrg[k];
        dr[k] = f1 * t0[k] + f2 * (t1[k] + t2[k] + t3[k]) + f3 * (t4[k] + t5[k]) + (clamped ? 0.f : dth * r[k] / th);
        dp[k] = f1 * gxr[k] + f2 * rrg[k];
    }
    if (bad) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { dr[k] = 0.f; dv[k] = 0.f; dp[k] = 0.f; }
    }
}

__global__ void __launch_bounds__(kVjpThreads, 1) deform_input_grad_kernel(const __grid_constant__ VjpKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemVjp &sm = *reinterpret_cast<SmemVjp *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int64_t n = K.S.n_samples_dev ? min(*K.S.n_samples_dev, K.S.n_samples) : K.S.n_samples;
    const int64_t n_tiles = (n + NSB_TILE - 1) / NSB_TILE;
    const int64_t my_tiles = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    {
        const uint4 *pe = reinterpret_cast<const uint4 *>(K.V.deform_packed_pe_t);
        for (int i = tid; i < 2 * kPeU4; i += kVjpThreads) (&sm.pe_t[0][0])[i] = __ldg(pe + i);
        for (int i = tid; i < 6 * 128 + 8; i += kVjpThreads) sm.bias[i] = K.P.deform_bias[i];
        if (tid == 0) {
            for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], 8); }
            mbar_fence_init();
        }
    }
    __syncthreads();
    const float ls = K.V.loss_scale, inv_ls = 1.0f / K.V.loss_scale;
    Ring rf;
    rf.producer = tid == 0;
    rf.total = (uint32_t)(my_tiles * kChunksPerTile);
    rf.fwd = reinterpret_cast<const uint8_t *>(K.P.deform_packed_tb);
    rf.bwd = reinterpret_cast<const uint8_t *>(K.V.deform_packed_t);
    rf.gbase = 0;
    for (uint32_t c = 0; c < kStages - 1; ++c) rf.issue(sm, c);
    __syncwarp();
    WarpScratch &ws = sm.ws[warp];
    const float amin[3] = {K.P.aabb[0], K.P.aabb[1], K.P.aabb[2]};
    const float *const gcb = K.S.sample_code_bias ? K.S.sample_code_bias : K.P.deform_code_bias;

#pragma unroll 1
    for (int64_t it = 0; it < my_tiles; ++it) {
        const int64_t tile = blockIdx.x + it * gridDim.x;
        const int64_t row0 = tile * NSB_TILE + warp * 16;
        rf.gbase = (uint32_t)(it * kChunksPerTile);
        __syncwarp();
        if (lane < 16) {   // one row per lane: the position and timestep exactly as the field kernels form them
            const int64_t s = row0 + lane;
            float px = 0.f, py = 0.f, pz = 0.f, tt = 0.f;
            if (s < n) {
                if (K.S.origins != nullptr) {
                    const int ri = K.S.ray_indices[s];
                    const float mid = __fadd_rn(K.S.t_starts[s], K.S.t_ends[s]);
                    px = ray_midpoint(K.S.origins[3 * (int64_t)ri + 0], K.S.directions[3 * (int64_t)ri + 0], mid);
                    py = ray_midpoint(K.S.origins[3 * (int64_t)ri + 1], K.S.directions[3 * (int64_t)ri + 1], mid);
                    pz = ray_midpoint(K.S.origins[3 * (int64_t)ri + 2], K.S.directions[3 * (int64_t)ri + 2], mid);
                    if (K.S.ray_times) tt = K.S.ray_times[ri];
                } else {
                    px = K.S.positions[3 * s + 0]; py = K.S.positions[3 * s + 1]; pz = K.S.positions[3 * s + 2];
                    if (K.S.sample_times) tt = K.S.sample_times[s];
                }
            }
            int tsi = sample_timestep(tt, K.P.n_timesteps);
            if (K.S.sample_code_bias) tsi = (int)min(s, n - 1);     // per-sample warp codes: the bias rows are per sample
            ws.pos[lane][0] = box_coord(px, amin[0], K.aabb_size[0]);
            ws.pos[lane][1] = box_coord(py, amin[1], K.aabb_size[1]);
            ws.pos[lane][2] = box_coord(pz, amin[2], K.aabb_size[2]);
            ws.pos[lane][3] = __int_as_float(tsi);
        }
        __syncwarp();
        float pn[2][3];    // rows g / g+8
        uint32_t cb[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            pn[h][0] = ws.pos[g + 8 * h][0]; pn[h][1] = ws.pos[g + 8 * h][1]; pn[h][2] = ws.pos[g + 8 * h][2];
            cb[h] = (uint32_t)__float_as_int(ws.pos[g + 8 * h][3]) * 256u;
        }
        // ---- forward: windowed posenc fragments (the field kernels' expressions) ----
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
                        e0 = wj * sinf(arg);
                        e1 = wj * sinf(arg + 1.5707963267948966f);
                    } else if (i == 21) {
                        e0 = kTwoPi * pn[h][0];
                        e1 = kTwoPi * pn[h][1];
                    } else if (i == 22) {
                        e0 = kTwoPi * pn[h][2];
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
        // ---- forward: six stem layers; m[l][half] = ReLU bits of layer l's output ----
        uint32_t m[6][2];
        float acc[8][4];
        zero8(acc); ring_gemm<3>(acc, kF_L0, in_a, sm, rf, lane); m[0][0] = relu_store<0, true>(acc, ws.act[0], nullptr, gcb, cb, q, lane);
        zero8(acc); ring_gemm<3>(acc, kF_L0 + 3, in_a, sm, rf, lane); m[0][1] = relu_store<1, true>(acc, ws.act[0], nullptr, gcb, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L1, buf0, sm, rf, lane); m[1][0] = relu_store<0, false>(acc, ws.act[1], sm.bias + 1 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L1 + 8, buf0, sm, rf, lane); m[1][1] = relu_store<1, false>(acc, ws.act[1], sm.bias + 1 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L2, buf1, sm, rf, lane); m[2][0] = relu_store<0, false>(acc, ws.act[0], sm.bias + 2 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L2 + 8, buf1, sm, rf, lane); m[2][1] = relu_store<1, false>(acc, ws.act[0], sm.bias + 2 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L3, buf0, sm, rf, lane); m[3][0] = relu_store<0, false>(acc, ws.act[1], sm.bias + 3 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L3 + 8, buf0, sm, rf, lane); m[3][1] = relu_store<1, false>(acc, ws.act[1], sm.bias + 3 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<11>(acc, kF_L4, skip_a, sm, rf, lane); m[4][0] = relu_store<0, true>(acc, ws.act[0], nullptr, gcb + 128, cb, q, lane);
        zero8(acc); ring_gemm<11>(acc, kF_L4 + 11, skip_a, sm, rf, lane); m[4][1] = relu_store<1, true>(acc, ws.act[0], nullptr, gcb + 128, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L5, buf0, sm, rf, lane); m[5][0] = relu_store<0, false>(acc, ws.act[1], sm.bias + 5 * 128, nullptr, cb, q, lane);
        zero8(acc); ring_gemm<8>(acc, kF_L5 + 8, buf0, sm, rf, lane); m[5][1] = relu_store<1, false>(acc, ws.act[1], sm.bias + 5 * 128, nullptr, cb, q, lane);
        // ---- forward heads: (v, r) of rows g / g+8.  First half of the split chunk; the transposed heads follow in it ----
        float hacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        {
            const uint32_t G = rf.gbase + kF_HEADS / kChunkSlabs;
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
        }
        const float hb0 = sm.bias[6 * 128 + 2 * q], hb1 = sm.bias[6 * 128 + 2 * q + 1];
        const float c0 = hacc[0][0] + hb0, c1 = hacc[0][1] + hb1, c2 = hacc[0][2] + hb0, c3 = hacc[0][3] + hb1;
        const int rsel = q & 1;
        float vr[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int srcl = (lane & ~3) | k;
            const float a0 = __shfl_sync(0xffffffffu, c0, srcl), a1 = __shfl_sync(0xffffffffu, c1, srcl);
            const float b0 = __shfl_sync(0xffffffffu, c2, srcl), b1 = __shfl_sync(0xffffffffu, c3, srcl);
            vr[2 * k] = rsel ? b0 : a0;
            vr[2 * k + 1] = rsel ? b1 : a1;
        }
        // ---- SE(3) backward of this lane's row (q = 0: row g, q = 1: row g+8) ----
        float dvr[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, direct[3] = {0.f, 0.f, 0.f};
        const int64_t srow = row0 + g + 8 * rsel;
        if (q < 2 && srow < n) {
            const float p[3] = {rsel ? pn[1][0] : pn[0][0], rsel ? pn[1][1] : pn[0][1], rsel ? pn[1][2] : pn[0][2]};
            const float v[3] = {vr[0], vr[1], vr[2]}, r[3] = {vr[3], vr[4], vr[5]};
            const float u[3] = {K.V.u[3 * srow + 0] * K.u_scale[0], K.V.u[3 * srow + 1] * K.u_scale[1],
                                K.V.u[3 * srow + 2] * K.u_scale[2]};
            float dr[3], dv[3];
            se3_input_vjp(p, r, v, u, dr, dv, direct);
            dvr[0] = dv[0]; dvr[1] = dv[1]; dvr[2] = dv[2]; dvr[3] = dr[0]; dvr[4] = dr[1]; dvr[5] = dr[2];
        }
        // (dv, dr) x loss scale as the A fragment of the heads' delta: lane q holds cols 2q, 2q+1 of rows g (from lane
        // 4g) and g+8 (from lane 4g+1); k 6..15 are padding
        uint32_t dAh[4] = {0u, 0u, 0u, 0u};
        {
            const int la = lane & ~3, lb = (lane & ~3) | 1;
            float ra[6], rb[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) { ra[k] = __shfl_sync(0xffffffffu, dvr[k], la); rb[k] = __shfl_sync(0xffffffffu, dvr[k], lb); }
            if (q < 3) {
                dAh[0] = pack_h2(ls * (q == 0 ? ra[0] : (q == 1 ? ra[2] : ra[4])), ls * (q == 0 ? ra[1] : (q == 1 ? ra[3] : ra[5])));
                dAh[1] = pack_h2(ls * (q == 0 ? rb[0] : (q == 1 ? rb[2] : rb[4])), ls * (q == 0 ? rb[1] : (q == 1 ? rb[3] : rb[5])));
            }
        }
        // ---- delta chain: delta_5 = (delta_heads . W_heads) * relu'(a5), then L5 .. L1 ----
        auto ah = [&](int, uint32_t(&a)[4]) { a[0] = dAh[0]; a[1] = dAh[1]; a[2] = dAh[2]; a[3] = dAh[3]; };
        zero8(acc); ring_gemm<1>(acc, kB_HEADS, ah, sm, rf, lane); delta_store<0>(acc, ws.act[0], m[5][0], lane);
        zero8(acc); ring_gemm<1>(acc, kB_HEADS + 1, ah, sm, rf, lane); delta_store<1>(acc, ws.act[0], m[5][1], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L5, buf0, sm, rf, lane); delta_store<0>(acc, ws.act[1], m[4][0], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L5 + 8, buf0, sm, rf, lane); delta_store<1>(acc, ws.act[1], m[4][1], lane);
        // d enc = delta_4 . W4[:, posenc] (skip connection) + delta_0 . W0[:, posenc]: 6 n-tiles of 8 kernel-order columns
        float pe[6][4];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) pe[i][k] = 0.f;
        auto pe_gemm = [&](const uint4 *wt, const uint4 (*src)[32]) {
#pragma unroll 2
            for (int kt = 0; kt < 8; ++kt) {
                const uint4 av = src[kt][lane];
                const uint32_t a[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                for (int p = 0; p < 3; ++p) {
                    const uint4 b = wt[(kt * 3 + p) * 32 + lane];
                    mma16816(pe[2 * p], a, b.x, b.y);
                    mma16816(pe[2 * p + 1], a, b.z, b.w);
                }
            }
        };
        pe_gemm(sm.pe_t[1], ws.act[1]);
        zero8(acc); ring_gemm<8>(acc, kB_L4H, buf1, sm, rf, lane); delta_store<0>(acc, ws.act[0], m[3][0], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L4H + 8, buf1, sm, rf, lane); delta_store<1>(acc, ws.act[0], m[3][1], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L3, buf0, sm, rf, lane); delta_store<0>(acc, ws.act[1], m[2][0], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L3 + 8, buf0, sm, rf, lane); delta_store<1>(acc, ws.act[1], m[2][1], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L2, buf1, sm, rf, lane); delta_store<0>(acc, ws.act[0], m[1][0], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L2 + 8, buf1, sm, rf, lane); delta_store<1>(acc, ws.act[0], m[1][1], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L1, buf0, sm, rf, lane); delta_store<0>(acc, ws.act[1], m[0][0], lane);
        zero8(acc); ring_gemm<8>(acc, kB_L1 + 8, buf0, sm, rf, lane); delta_store<1>(acc, ws.act[1], m[0][1], lane);
        pe_gemm(sm.pe_t[0], ws.act[1]);
        // ---- posenc backward: this lane holds (d sin_i, d cos_i) of argument i = 4 nt + q for rows g (0, 1) / g+8 (2, 3) ----
        float dp[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
        for (int nt = 0; nt < 6; ++nt) {
            const int i = nt * 4 + q;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float d0 = pe[nt][2 * h], d1 = pe[nt][2 * h + 1];
                if (i < 21) {
                    const int d = i / 7, j = i - d * 7;
                    const float pd = d == 0 ? pn[h][0] : (d == 1 ? pn[h][1] : pn[h][2]);
                    const float fr = kTwoPi * (float)(1 << j);
                    float sn, cs;
                    sincosf((kTwoPi * pd) * (float)(1 << j), &sn, &cs);
                    const float val = (K.O.pe_window[j] * fr) * (cs * d0 - sn * d1);
                    dp[h][0] += d == 0 ? val : 0.f; dp[h][1] += d == 1 ? val : 0.f; dp[h][2] += d == 2 ? val : 0.f;
                } else if (i == 21) {
                    dp[h][0] += kTwoPi * d0; dp[h][1] += kTwoPi * d1;
                } else if (i == 22) {
                    dp[h][2] += kTwoPi * d0;
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                dp[h][k] += __shfl_xor_sync(0xffffffffu, dp[h][k], 1);
                dp[h][k] += __shfl_xor_sync(0xffffffffu, dp[h][k], 2);
            }
        if (q < 2 && srow < n) {
#pragma unroll
            for (int k = 0; k < 3; ++k) K.V.d_pn[3 * srow + k] = (rsel ? dp[1][k] : dp[0][k]) * inv_ls + direct[k];
        }
    }
}

}  // namespace

int launch_deform_input_grad(const char *who, const nsb_field_params *params, const nsb_field_opts *opts,
                             const nsb_samples *samples, const nsb_deform_vjp_args *args, const float u_scale[3],
                             cudaStream_t st) {
    if (!args->deform_packed_t || !args->deform_packed_pe_t || !args->u || !args->d_pn || !params->deform_packed_tb ||
        !params->deform_bias || (!params->deform_code_bias && !samples->sample_code_bias) || !(args->loss_scale > 0.f)) {
        set_error("%s: deformation input gradient: missing tensors", who);
        return 1;
    }
    if (samples->sample_code_bias && samples->n_samples > ((int64_t)1 << 24)) {
        set_error("%s: per-sample code bias: at most 2^24 samples", who);
        return 1;
    }
    VjpKArgs K;
    K.P = *params; K.O = *opts; K.S = *samples; K.V = *args;
    for (int k = 0; k < 3; ++k) { K.aabb_size[k] = params->aabb[3 + k] - params->aabb[k]; K.u_scale[k] = u_scale[k]; }
    const int smem = (int)sizeof(SmemVjp);
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(deform_input_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(deform_input_grad_kernel): %s", cudaGetErrorString(e)); return 1; }
        configured = true;
    }
    const int64_t n_tiles = (samples->n_samples + NSB_TILE - 1) / NSB_TILE;
    const int n_ctas = (int)std::min<int64_t>(n_tiles, num_sms());
    deform_input_grad_kernel<<<n_ctas, kVjpThreads, smem, st>>>(K);
    return check_launch("deform_input_grad_kernel");
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_deform_input_grad(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                     const nsb_deform_vjp_args *args, void *stream) {
    if (!params || !opts || !samples || !args) { set_error("nsb_deform_input_grad: null argument"); return 1; }
    if (check_field_params("nsb_deform_input_grad", params) || check_samples("nsb_deform_input_grad", samples)) return 1;
    if (samples->n_samples <= 0) return 0;
    const float one[3] = {1.f, 1.f, 1.f};
    return launch_deform_input_grad("nsb_deform_input_grad", params, opts, samples, args, one, (cudaStream_t)stream);
}
