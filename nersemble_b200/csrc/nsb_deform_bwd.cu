// Backward of the SE(3) deformation field (training), sm_90a.
//
// Replaces the autograd of (reference, relative to /root/reference/src/nersemble/):
//   nerfstudio/field_components/deformation_field.py:77-116,148-166   mlp_stem / mlp_r / mlp_v, offsets
//   util/pytorch3d.py:107-191                                          se3_exp_map
//   nerfstudio/models/nersemble_instant_ngp.py:120-125,315             time_embedding_deformation (warp codes)
//
// One CTA = 8 warps = one 128-sample tile; warp w owns rows 16w..16w+15 for the delta chain.
//   * stem activations come from the training forward (nsb_field_out.deform_acts / deform_enc, A-fragment
//     order) -- nothing is recomputed except the tiny heads GEMM that reproduces (v, r);
//   * SE(3) exp-map backward in fp32 per row, then deltas flow back through the six layers on mma.sync with
//     TRANSPOSED weight fragments streamed from L2 through the same cp.async.bulk/mbarrier ring as the forward;
//   * weight gradients dW_l = delta_l^T . a_{l-1} are reduced over all 128 rows of the tile before touching
//     memory: every warp stages its delta / activation fragments in shared memory, then warp w computes the
//     output-row block w of dW_l (movmatrix transposes, K = 8 row blocks) and adds it to the fp32 gradient;
//   * warp-code gradients = delta . W[:, code columns], summed over the rows of a warp (one ray -> one timestep).
#include <algorithm>
#include <cstddef>
#include <cstring>
#include <type_traits>

#include "nsb_common.cuh"

namespace nsb {

// nsb_deform_bwd_args without its trailing per-sample-code fields: the table-code kernel keeps its parameter offsets
// (aabb_size follows B), the per-sample pointers ride after aabb_size in DeformBwdKArgsPS.
struct DeformBwdCore {
    const void *deform_packed_t, *deform_acts, *deform_enc;
    const float *d_xs;
    float loss_scale;
    float *d_stem_w[6];
    float *d_stem_b, *d_r_w, *d_r_b, *d_v_w, *d_v_b, *d_warp_codes;
    void *dw_workspace;
};
static_assert(sizeof(DeformBwdCore) == offsetof(nsb_deform_bwd_args, sample_warp_codes) &&
              offsetof(DeformBwdCore, loss_scale) == offsetof(nsb_deform_bwd_args, loss_scale) &&
              offsetof(DeformBwdCore, d_stem_w) == offsetof(nsb_deform_bwd_args, d_stem_w) &&
              offsetof(DeformBwdCore, dw_workspace) == offsetof(nsb_deform_bwd_args, dw_workspace),
              "DeformBwdCore must be the leading part of nsb_deform_bwd_args");

struct DeformBwdKArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    DeformBwdCore B;
    float aabb_size[3];
};
struct DeformBwdKArgsPS : DeformBwdKArgs {
    const __half *sample_warp_codes;   // [n][128]
    float *d_sample_warp_codes;        // [n][128] or NULL
};
template <bool PER_SAMPLE>
using DeformBwdKArgsT = std::conditional_t<PER_SAMPLE, DeformBwdKArgsPS, DeformBwdKArgs>;

constexpr int kDSlab = 2048, kDChunkSlabs = 4, kDChunkBytes = kDSlab * kDChunkSlabs, kDStages = 4;
// transposed slab order = order of use: heads, L5, L4 (hidden cols), L4 (code cols), L3, L2, L1, L0 (code cols)
constexpr int jT_HEADS = 0, jT_L5 = 2, jT_L4H = 18, jT_L4C = 34, jT_L3 = 50, jT_L2 = 66, jT_L1 = 82, jT_L0C = 98;
constexpr int kTSlabs = 114;
constexpr int kTChunks = (kTSlabs + kDChunkSlabs - 1) / kDChunkSlabs;   // 29

struct alignas(128) SmemDB {
    uint8_t ring[kDStages][kDChunkBytes];
    uint64_t full[kDStages], empty[kDStages];
    uint4 heads_w[8 * 32];        // forward heads fragments (8 k-tiles x 1 pair)
    float bias_heads[8];
    int ts[NSB_TILE];
    uint4 D[8][8][32];            // delta fragments of every warp (A-fragment order, 8 k-tiles of 16 outputs)
    uint4 X[8][19][32];           // layer-input fragments of every warp, TRANSPOSED (movmatrix): [hidden 8 | enc 3 | code 8]
    float bias_acc[6][128];       // per-CTA bias-gradient accumulator (x loss scale), flushed once at the end
};

__device__ __forceinline__ uint32_t movt(uint32_t a) {
    uint32_t d;
    asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
    return d;
}

__device__ __forceinline__ uint4 movt4(const uint4 v) { return make_uint4(movt(v.x), movt(v.y), movt(v.z), movt(v.w)); }

// bit e of the result: element e (low/high half of x, y, z, w) of the fragment is > 0   (ReLU derivative of a saved activation)
__device__ __forceinline__ uint32_t pos_bits(const uint4 v) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        // activations are post-ReLU fp16 (>= 0, never -0 from fmaxf(x, 0)): "> 0" is "bits != 0"
        m |= ((w[k] & 0xffffu) != 0u ? 1u : 0u) << (2 * k);
        m |= ((w[k] >> 16) != 0u ? 1u : 0u) << (2 * k + 1);
    }
    return m;
}

struct TRing {
    bool producer;
    uint32_t gbase, total;
    const uint8_t *src;
    __device__ __forceinline__ void issue(SmemDB &sm, uint32_t gt) const {
        if (producer && gt < total) {
            const uint32_t s = gt % kDStages, kf = gt / kDStages, c = gt % kTChunks;
            mbar_wait<20>(&sm.empty[s], (kf & 1) ^ 1);
            const uint32_t bytes = (c == kTChunks - 1) ? (kTSlabs - c * kDChunkSlabs) * kDSlab : kDChunkBytes;
            mbar_expect_tx(&sm.full[s], bytes);
            bulk_g2s(sm.ring[s], src + (size_t)c * kDChunkBytes, bytes, &sm.full[s]);
        }
    }
};

// acc[8][4] += A(16 x 16*KT) . slabs j0..j0+KT-1 (one N-half of 64 columns each)
template <class AFn>
__device__ __forceinline__ void tring_gemm(float (&acc)[8][4], const int j0, const int KT, AFn &&afn, SmemDB &sm,
                                           const TRing &rf, int lane) {
#pragma unroll 2
    for (int kt = 0; kt < KT; ++kt) {
        const int j = j0 + kt;
        const uint32_t G = rf.gbase + (j >> 2);
        const int stage = G & 3;
        if ((j & 3) == 0) {
            rf.issue(sm, G + (kDStages - 1));
            __syncwarp();
            mbar_wait<20>(&sm.full[stage], (G >> 2) & 1);
        }
        uint32_t a[4];
        afn(kt, a);
        const uint4 *slab = reinterpret_cast<const uint4 *>(&sm.ring[stage][(j & 3) * kDSlab]);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const uint4 b = slab[p * 32 + lane];
            mma16816(acc[2 * p], a, b.x, b.y);
            mma16816(acc[2 * p + 1], a, b.z, b.w);
        }
        if ((j & 3) == 3 || j == kTSlabs - 1) {
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

__device__ __forceinline__ void cross(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// backward of pw = R(r) p + V(r) v  (util/pytorch3d.py:107-191 + deformation_field.py:95-107); g = dL/dpw
__device__ __forceinline__ void se3_backward(const float p[3], const float r[3], const float v[3], const float g[3],
                                             float dr[3], float dv[3]) {
    const float n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    const bool clamped = !(n2 > 1e-4f);
    const float th = sqrtf(fmaxf(n2, 1e-4f));
    float s, c;
    sincosf(th, &s, &c);
    const float th2 = th * th;
    const float f1 = s / th, f2 = (1.0f - c) / th2, f3 = (th - s) / (th2 * th);
    float A[3], Bv[3], Cv[3], Dv[3], gxr[3], rxg[3], rrg[3], t0[3], t1[3], t2[3], t3[3], t4[3];
    cross(r, p, A); cross(r, A, Bv); cross(r, v, Cv); cross(r, Cv, Dv);
    cross(g, r, gxr); cross(r, g, rxg); cross(r, rxg, rrg);
    cross(p, g, t0);      // d/dr [g.(r x p)]
    cross(A, g, t1);      // d/dr [g.(r x u)], u = r x p fixed
    cross(p, gxr, t2);    //   ... through u
    cross(v, g, t3);      // d/dr [g.(r x v)]
    cross(Cv, g, t4);     // d/dr [g.(r x w)], w = r x v fixed
    float t5[3];
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
    }
    if (bad) {   // NaN warp -> identity (deformation_field.py:101-102): no gradient
#pragma unroll
        for (int k = 0; k < 3; ++k) { dr[k] = 0.f; dv[k] = 0.f; }
    }
}

// kernel posenc column k' (0..47) -> column of the reference's layer input (or -1)
__device__ __forceinline__ int enc_ref_col(int kp) {
    const int i = kp >> 1, s = kp & 1;
    if (i < 21) return s == 0 ? i : 21 + i;
    if (i == 21) return 42 + s;
    if (i == 22) return s == 0 ? 44 : -1;
    return -1;
}

// ---------------------------------------------------------------------------------------------
// Weight-gradient accumulation.  First version: every tile added its dW block to the fp32 gradient with atomicAdd --
// 127 K atomics per 128-row tile, 1.8 G per step on ~126 K hot addresses: the kernel's bottleneck.  Now each
// CTA owns a private fp32 accumulator in FRAGMENT order (workspace [cta][kScrF4] float4): a lane adds its MMA
// accumulators to its own float4 slots -- coalesced 512 B per warp access, no atomics, L2-resident (0.5 MB per CTA) --
// and deform_dw_reduce_kernel sums the CTAs' accumulators into the reference layout once at the end.
// Site layout per CTA (float4 units): [warp/ob 8][NIB][h 2][lane 32].
// ---------------------------------------------------------------------------------------------
constexpr int kSiteL5 = 0, kSiteL4A = 4096, kSiteL4B = 8192, kSiteL3 = 13824, kSiteL2 = 17920, kSiteL1 = 22016,
              kSiteL0 = 26112, kScrF4 = 31744;

// dW block: output rows 16*ob.., input k-tiles IB0..IB0+NIB-1 of X, reduced over the 8 row blocks of the tile.
// sm.X holds the input fragments already TRANSPOSED (each warp transposes its own block once when staging; before,
// all 8 warps repeated the movmatrix of every block: 262 M MOVM per step, more than the HMMAs).
// BIAS: the bias gradient (column sums of delta) rides along as one more HMMA per row block against an all-ones B
// fragment; lane (g, q == 0) owns outputs 16*ob + g and + 8 of bias_acc (no shuffles, no atomics).
// NTOT / I0: the site holds NTOT input k-tiles per output block; this call covers tiles I0..I0+NIB-1 of them (wide
// layers are done in two calls: 11 k-tiles of accumulators would be 88 registers of the 128 a 512-thread CTA allows).
template <int IB0, int NIB, bool BIAS, int NTOT = NIB, int I0 = 0>
__device__ __forceinline__ void dw_slice(SmemDB &sm, int ob, float4 *site, bool first, float *bias_acc, int lane) {
    float acc[NIB][2][4];
    float bsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NIB; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][h][k] = 0.f;
#pragma unroll 1
    for (int rb = 0; rb < 8; ++rb) {
        const uint4 d = sm.D[rb][ob][lane];
        const uint32_t a[4] = {movt(d.x), movt(d.z), movt(d.y), movt(d.w)};   // delta^T block (see nsb_backward.cu)
        if (BIAS) mma16816(bsum, a, 0x3c003c00u, 0x3c003c00u);                // x ones: every column = sum over the 16 rows
#pragma unroll
        for (int i = 0; i < NIB; ++i) {
            const uint4 x = sm.X[rb][IB0 + i][lane];
            mma16816(acc[i][0], a, x.x, x.y);
            mma16816(acc[i][1], a, x.z, x.w);
        }
    }
    if (BIAS && (lane & 3) == 0) {
        bias_acc[ob * 16 + (lane >> 2)] += bsum[0];
        bias_acc[ob * 16 + (lane >> 2) + 8] += bsum[2];
    }
    float4 *dst = site + (size_t)ob * NTOT * 64 + I0 * 64 + lane;
    if (first) {
#pragma unroll
        for (int i = 0; i < NIB; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) dst[(i * 2 + h) * 32] = make_float4(acc[i][h][0], acc[i][h][1], acc[i][h][2], acc[i][h][3]);
    } else {
        // fire-and-forget vector reductions: nobody else touches these lines, and unlike load-add-store the warp does
        // not wait a DRAM/L2 round trip per slice (the accumulators do not stay L2-resident next to 2.8 GB of streamed
        // activations)
#pragma unroll
        for (int i = 0; i < NIB; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + (i * 2 + h) * 32), "f"(acc[i][h][0]),
                             "f"(acc[i][h][1]), "f"(acc[i][h][2]), "f"(acc[i][h][3]) : "memory");
    }
}

// sums the CTAs' fragment-order accumulators into the reference layouts (nn.Linear weight [out][in], += , x 1/loss_scale)
struct DwReduceArgs {
    const float4 *scratch;
    int n_ctas;
    float inv_ls;
    float *d_stem_w[6];
};
__global__ void __launch_bounds__(256) deform_dw_reduce_kernel(const __grid_constant__ DwReduceArgs R) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= kScrF4) return;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < R.n_ctas; ++c) {
        const float4 v = __ldg(R.scratch + (size_t)c * kScrF4 + idx);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    int layer, ib0, nib, ld, base;
    if (idx < kSiteL4A) { layer = 5; ib0 = 0; nib = 8; ld = 128; base = kSiteL5; }
    else if (idx < kSiteL4B) { layer = 4; ib0 = 0; nib = 8; ld = 301; base = kSiteL4A; }
    else if (idx < kSiteL3) { layer = 4; ib0 = 8; nib = 11; ld = 301; base = kSiteL4B; }
    else if (idx < kSiteL2) { layer = 3; ib0 = 0; nib = 8; ld = 128; base = kSiteL3; }
    else if (idx < kSiteL1) { layer = 2; ib0 = 0; nib = 8; ld = 128; base = kSiteL2; }
    else if (idx < kSiteL0) { layer = 1; ib0 = 0; nib = 8; ld = 128; base = kSiteL1; }
    else { layer = 0; ib0 = 0; nib = 11; ld = 173; base = kSiteL0; }
    const int r = idx - base, lane = r & 31, h = (r >> 5) & 1, i = (r >> 6) % nib, ob = (r >> 6) / nib;
    const int g = lane >> 2, q = lane & 3;
    const int o = ob * 16 + g, kc = (ib0 + i) * 16 + h * 8 + 2 * q;
    auto col_of = [&](int k) -> int {
        if (layer == 4) { if (k < 128) return 173 + k; const int kk = k - 128; return kk < 48 ? enc_ref_col(kk) : 45 + (kk - 48); }
        if (layer == 0) return k < 48 ? enc_ref_col(k) : 45 + (k - 48);
        return k;
    };
    float *dw = R.d_stem_w[layer];
    const int c0 = col_of(kc), c1 = col_of(kc + 1);
    if (c0 >= 0) { dw[(size_t)o * ld + c0] += s.x * R.inv_ls; dw[(size_t)(o + 8) * ld + c0] += s.z * R.inv_ls; }
    if (c1 >= 0) { dw[(size_t)o * ld + c1] += s.y * R.inv_ls; dw[(size_t)(o + 8) * ld + c1] += s.w * R.inv_ls; }
}

// 16 warps, two roles that only meet at the per-layer barriers:
//   CHAIN warps 0-7  : rows 16w..16w+15 -- SE(3) backward, delta chain through the transposed weights (ring), staging
//   DW    warps 8-15 : output block ob = w - 8 of every weight gradient (tile-wide contraction), bias sums
// (One role per warp doubled the resident warps: the 8-warp version was latency-bound at
//  12.5 % occupancy, the dX chain and the dW contraction of a layer are independent once D / X are staged.)
// PER_SAMPLE: the warp codes are per-sample rows (component API) instead of the timestep's row of the embedding, and the
// code-column gradient of every row is written to its own row of d_sample_warp_codes.
constexpr int kDbThreads = 512;
template <bool PER_SAMPLE>
__global__ void __launch_bounds__(kDbThreads, 1) deform_bwd_kernel(const __grid_constant__ DeformBwdKArgsT<PER_SAMPLE> K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemDB &sm = *reinterpret_cast<SmemDB *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31;
    const bool chain = tid < 256;
    const int warp = (tid >> 5) & 7;          // CHAIN: row block; DW: output block
    const int g = lane >> 2, q = lane & 3;
    const int64_t n = K.S.n_samples;
    const int64_t n_tiles = (n + NSB_TILE - 1) / NSB_TILE;
    const int64_t my_tiles = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    {   // forward heads fragments live at the end of deform_packed_tb (slabs 92,93 of 94)
        const uint4 *hw = reinterpret_cast<const uint4 *>(reinterpret_cast<const uint8_t *>(K.P.deform_packed_tb) + 92 * 2048);
        for (int i = tid; i < 256; i += kDbThreads) sm.heads_w[i] = __ldg(hw + i);
        if (tid < 8) sm.bias_heads[tid] = K.P.deform_bias[6 * 128 + tid];
        for (int i = tid; i < 6 * 128; i += kDbThreads) (&sm.bias_acc[0][0])[i] = 0.f;
        if (tid == 0) {
            for (int s = 0; s < kDStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], 8); }
            mbar_fence_init();
        }
    }
    __syncthreads();
    const float ls = K.B.loss_scale, inv_ls = 1.0f / K.B.loss_scale;
    TRing rf;
    rf.producer = tid == 0;
    rf.total = (uint32_t)(my_tiles * kTChunks);
    rf.src = reinterpret_cast<const uint8_t *>(K.B.deform_packed_t);
    rf.gbase = 0;
    if (chain) {
        for (uint32_t c = 0; c < kDStages - 1; ++c) rf.issue(sm, c);
        __syncwarp();
    }
    const uint4 *acts = reinterpret_cast<const uint4 *>(K.B.deform_acts);
    const uint4 *encs = reinterpret_cast<const uint4 *>(K.B.deform_enc);
    const float amin[3] = {K.P.aabb[0], K.P.aabb[1], K.P.aabb[2]};
    float4 *scr = reinterpret_cast<float4 *>(K.B.dw_workspace) + (size_t)blockIdx.x * kScrF4;

    for (int64_t it = 0; it < my_tiles; ++it) {
        const int64_t tile = blockIdx.x + it * gridDim.x;
        const int64_t row0 = tile * NSB_TILE + warp * 16;
        rf.gbase = (uint32_t)(it * kTChunks);
        const uint4 *act_w = acts + ((size_t)tile * 8 + warp) * 6 * 256;     // [layer][kt][lane]
        const uint4 *enc_w = encs + ((size_t)tile * 8 + warp) * 3 * 32;
        int tsr[2] = {0, 0};
        bool ts_uniform = true;
        uint32_t dAh[4] = {0u, 0u, 0u, 0u};
        uint32_t relu_lo = 0, relu_hi = 0;     // ReLU-derivative bits of the staged activation: k-tiles 0-3 / 4-7, 8 bits each
        uint32_t dcur[8][4];
        if (chain) {
        // ---- per-row inputs: normalised position and timestep of rows g / g+8 ----
        float pn[2][3];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t s = row0 + g + 8 * h;
            float px = 0.f, py = 0.f, pz = 0.f, tt = 0.f;
            if (s < n) {
                if (K.S.origins != nullptr) {
                    const int ri = K.S.ray_indices[s];
                    const float mid = __fadd_rn(K.S.t_starts[s], K.S.t_ends[s]);
                    px = __fadd_rn(K.S.origins[3 * (int64_t)ri + 0], __fmul_rn(__fmul_rn(K.S.directions[3 * (int64_t)ri + 0], mid), 0.5f));
                    py = __fadd_rn(K.S.origins[3 * (int64_t)ri + 1], __fmul_rn(__fmul_rn(K.S.directions[3 * (int64_t)ri + 1], mid), 0.5f));
                    pz = __fadd_rn(K.S.origins[3 * (int64_t)ri + 2], __fmul_rn(__fmul_rn(K.S.directions[3 * (int64_t)ri + 2], mid), 0.5f));
                    if (K.S.ray_times) tt = K.S.ray_times[ri];
                } else {
                    px = K.S.positions[3 * s + 0]; py = K.S.positions[3 * s + 1]; pz = K.S.positions[3 * s + 2];
                    if (K.S.sample_times) tt = K.S.sample_times[s];
                }
            }
            pn[h][0] = __fdiv_rn(__fsub_rn(px, amin[0]), K.aabb_size[0]);
            pn[h][1] = __fdiv_rn(__fsub_rn(py, amin[1]), K.aabb_size[1]);
            pn[h][2] = __fdiv_rn(__fsub_rn(pz, amin[2]), K.aabb_size[2]);
            int t = __float2int_rn(__fmul_rn(tt, (float)(K.P.n_timesteps - 1)));
            tsr[h] = min(max(t, 0), K.P.n_timesteps - 1);
        }
        if (q == 0) { sm.ts[warp * 16 + g] = tsr[0]; sm.ts[warp * 16 + g + 8] = tsr[1]; }
        const int ts_lane0 = __shfl_sync(0xffffffffu, tsr[0], 0);   // (no shuffle inside a short-circuit expression)
        ts_uniform = __all_sync(0xffffffffu, (tsr[0] == ts_lane0) & (tsr[1] == ts_lane0));
        // ---- heads forward (v, r) from a5, SE(3) backward ----
        float hacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
        for (int kt = 0; kt < 8; ++kt) {
            const uint4 av = __ldcs(act_w + 5 * 256 + kt * 32 + lane);
            const uint32_t a[4] = {av.x, av.y, av.z, av.w};
            const uint4 b = sm.heads_w[kt * 32 + lane];
            mma16816(hacc[0], a, b.x, b.y);
            mma16816(hacc[1], a, b.z, b.w);
        }
        const float hb0 = sm.bias_heads[2 * q], hb1 = sm.bias_heads[2 * q + 1];
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
        float dvr[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // (dv, dr) of this lane's row (q=0: row g, q=1: row g+8)
        {
            const int64_t s = row0 + g + 8 * rsel;
            if (q < 2 && s < n) {
                const float p[3] = {rsel ? pn[1][0] : pn[0][0], rsel ? pn[1][1] : pn[0][1], rsel ? pn[1][2] : pn[0][2]};
                const float v[3] = {vr[0], vr[1], vr[2]}, r[3] = {vr[3], vr[4], vr[5]};
                // x_hash = ((p_world + offset) - aabb_min) / size with offset = pw - p in NORMALISED units (reference quirk)
                const float gp[3] = {K.B.d_xs[3 * s + 0] / K.aabb_size[0], K.B.d_xs[3 * s + 1] / K.aabb_size[1],
                                     K.B.d_xs[3 * s + 2] / K.aabb_size[2]};
                float dr[3], dv[3];
                se3_backward(p, r, v, gp, dr, dv);
                dvr[0] = dv[0]; dvr[1] = dv[1]; dvr[2] = dv[2]; dvr[3] = dr[0]; dvr[4] = dr[1]; dvr[5] = dr[2];
            }
        }
        // scatter (dv, dr) into accumulator layout: lane q holds cols 2q,2q+1 of rows g (from lane 4g) and g+8 (lane 4g+1)
        float dh[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        {
            const int la = lane & ~3, lb = (lane & ~3) | 1;
            float ra[6], rbv[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) { ra[k] = __shfl_sync(0xffffffffu, dvr[k], la); rbv[k] = __shfl_sync(0xffffffffu, dvr[k], lb); }
            if (q < 3) {
                dh[0][0] = ls * (q == 0 ? ra[0] : (q == 1 ? ra[2] : ra[4]));
                dh[0][1] = ls * (q == 0 ? ra[1] : (q == 1 ? ra[3] : ra[5]));
                dh[0][2] = ls * (q == 0 ? rbv[0] : (q == 1 ? rbv[2] : rbv[4]));
                dh[0][3] = ls * (q == 0 ? rbv[1] : (q == 1 ? rbv[3] : rbv[5]));
            }
            // bias gradients of mlp_v / mlp_r: column sums over the warp's 16 rows
            float s0 = dh[0][0] + dh[0][2], s1 = dh[0][1] + dh[0][3];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
            if (g == 0 && q < 3) {
                const int col = 2 * q;   // cols 0..2 = v, 3..5 = r
                float *b0p = col < 3 ? K.B.d_v_b + col : K.B.d_r_b + (col - 3);
                float *b1p = (col + 1) < 3 ? K.B.d_v_b + col + 1 : K.B.d_r_b + (col + 1 - 3);
                if (s0 != 0.f) atomicAdd(b0p, s0 * inv_ls);
                if (s1 != 0.f) atomicAdd(b1p, s1 * inv_ls);
            }
        }
        dAh[0] = pack_h2(dh[0][0], dh[0][1]); dAh[1] = pack_h2(dh[0][2], dh[0][3]);
        // ---- dW heads: stage delta (k-tile 0) and a5; DW warp ob takes one 16-column block of the 128 inputs ----
        sm.D[warp][0][lane] = make_uint4(dAh[0], dAh[1], dAh[2], dAh[3]);
#pragma unroll
        for (int kt = 0; kt < 8; ++kt) {
            const uint4 v = __ldcs(act_w + 5 * 256 + kt * 32 + lane);
            if (kt < 4) relu_lo |= pos_bits(v) << (8 * kt); else relu_hi |= pos_bits(v) << (8 * (kt - 4));
            sm.X[warp][kt][lane] = movt4(v);
        }
        }   // chain
        __syncthreads();
        if (!chain) {
            float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll 1
            for (int rb = 0; rb < 8; ++rb) {
                const uint4 d = sm.D[rb][0][lane];
                const uint32_t a[4] = {movt(d.x), movt(d.z), movt(d.y), movt(d.w)};
                const uint4 x = sm.X[rb][warp][lane];
                mma16816(acc[0], a, x.x, x.y);
                mma16816(acc[1], a, x.z, x.w);
            }
            // rows o = g (0..7) of the 16-row head block: 0..2 = mlp_v rows, 3..5 = mlp_r rows (rows 6..15 are padding)
            if (g < 6) {
                float *base = g < 3 ? K.B.d_v_w + g * 128 : K.B.d_r_w + (g - 3) * 128;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int col = warp * 16 + h * 8 + 2 * q;
                    atomicAdd(base + col, acc[h][0] * inv_ls);
                    atomicAdd(base + col + 1, acc[h][1] * inv_ls);
                }
            }
        }
        // ---- delta_5 = (delta_heads . W_heads) * (a5 > 0) ----
        if (chain) {
            auto ah = [&](int, uint32_t(&a)[4]) { a[0] = dAh[0]; a[1] = dAh[1]; a[2] = dAh[2]; a[3] = dAh[3]; };
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float acc[8][4];
                zero8(acc);
                tring_gemm(acc, jT_HEADS + half, 1, ah, sm, rf, lane);
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const int kt = half * 4 + nt / 2, rr = (nt & 1) * 2;
                    // fragment register rr (row g) / rr+1 (row g+8) of k-tile kt: bits 2*rr.. of its byte
                    const uint32_t mb = ((half == 0 ? relu_lo : relu_hi) >> (8 * (nt / 2) + 2 * rr)) & 0xfu;
                    dcur[kt][rr] = pack_h2(mb & 1u ? acc[nt][0] : 0.f, mb & 2u ? acc[nt][1] : 0.f);
                    dcur[kt][rr + 1] = pack_h2(mb & 4u ? acc[nt][2] : 0.f, mb & 8u ? acc[nt][3] : 0.f);
                }
            }
        }
        __syncthreads();   // everyone is done reading D/X of the heads step

        // ---- the six stem layers, last to first ----
#pragma unroll 1
        for (int l = 5; l >= 0; --l) {
            const bool has_hidden = l >= 1, has_in = (l == 4 || l == 0);
            if (chain) {
            // stage this layer's delta and input fragments
#pragma unroll
            for (int kt = 0; kt < 8; ++kt) sm.D[warp][kt][lane] = make_uint4(dcur[kt][0], dcur[kt][1], dcur[kt][2], dcur[kt][3]);
            if (has_hidden) {
                relu_lo = 0; relu_hi = 0;
#pragma unroll
                for (int kt = 0; kt < 8; ++kt) {
                    const uint4 v = __ldcs(act_w + (l - 1) * 256 + kt * 32 + lane);
                    if (kt < 4) relu_lo |= pos_bits(v) << (8 * kt); else relu_hi |= pos_bits(v) << (8 * (kt - 4));
                    sm.X[warp][kt][lane] = movt4(v);
                }
            }
            if (has_in) {
                const int eb = l == 4 ? 8 : 0;   // k-tile offset of [enc | code] inside X
#pragma unroll
                for (int kt = 0; kt < 3; ++kt) sm.X[warp][eb + kt][lane] = movt4(__ldcs(enc_w + kt * 32 + lane));
                if constexpr (PER_SAMPLE) {
                    // rows past the end stage zeros: their deltas are 0, and 0 x (uninitialised fp16) could be NaN
                    const int64_t sa = row0 + g, sb = row0 + g + 8;
                    const __half *cd0 = K.sample_warp_codes + (size_t)sa * NSB_WARP_CODE_DIM;
                    const __half *cd1 = K.sample_warp_codes + (size_t)sb * NSB_WARP_CODE_DIM;
#pragma unroll
                    for (int kc = 0; kc < 8; ++kc) {
                        uint4 cv = make_uint4(0u, 0u, 0u, 0u);
                        if (sa < n) {
                            cv.x = __ldg(reinterpret_cast<const uint32_t *>(cd0 + kc * 16 + 2 * q));
                            cv.z = __ldg(reinterpret_cast<const uint32_t *>(cd0 + kc * 16 + 2 * q + 8));
                        }
                        if (sb < n) {
                            cv.y = __ldg(reinterpret_cast<const uint32_t *>(cd1 + kc * 16 + 2 * q));
                            cv.w = __ldg(reinterpret_cast<const uint32_t *>(cd1 + kc * 16 + 2 * q + 8));
                        }
                        sm.X[warp][eb + 3 + kc][lane] = movt4(cv);
                    }
                } else {
                    const __half *cd0 = reinterpret_cast<const __half *>(K.P.warp_codes) + (size_t)tsr[0] * NSB_WARP_CODE_DIM;
                    const __half *cd1 = reinterpret_cast<const __half *>(K.P.warp_codes) + (size_t)tsr[1] * NSB_WARP_CODE_DIM;
#pragma unroll
                    for (int kc = 0; kc < 8; ++kc) {
                        uint4 cv;
                        cv.x = __ldg(reinterpret_cast<const uint32_t *>(cd0 + kc * 16 + 2 * q));
                        cv.y = __ldg(reinterpret_cast<const uint32_t *>(cd1 + kc * 16 + 2 * q));
                        cv.z = __ldg(reinterpret_cast<const uint32_t *>(cd0 + kc * 16 + 2 * q + 8));
                        cv.w = __ldg(reinterpret_cast<const uint32_t *>(cd1 + kc * 16 + 2 * q + 8));
                        sm.X[warp][eb + 3 + kc][lane] = movt4(cv);
                    }
                }
            }
            }   // chain: staging
            __syncthreads();
            // weight gradient: DW warp ob computes output rows 16ob..16ob+15 of dW_l
            if (!chain) {
            if (l == 4) {
                dw_slice<0, 8, true>(sm, warp, scr + kSiteL4A, it == 0, sm.bias_acc[4], lane);
                dw_slice<8, 6, false, 11, 0>(sm, warp, scr + kSiteL4B, it == 0, nullptr, lane);
                dw_slice<14, 5, false, 11, 6>(sm, warp, scr + kSiteL4B, it == 0, nullptr, lane);
            } else if (l == 0) {
                dw_slice<0, 6, true, 11, 0>(sm, warp, scr + kSiteL0, it == 0, sm.bias_acc[0], lane);
                dw_slice<6, 5, false, 11, 6>(sm, warp, scr + kSiteL0, it == 0, nullptr, lane);
            } else {
                const int site = l == 5 ? kSiteL5 : (l == 3 ? kSiteL3 : (l == 2 ? kSiteL2 : kSiteL1));
                dw_slice<0, 8, true>(sm, warp, scr + site, it == 0, sm.bias_acc[l], lane);
            }
            }   // DW warps
            // delta of the previous layer (own rows) and warp-code gradients, transposed weights from the ring
            // (A fragments come from the staged copy: a runtime k index into the register array would go to local memory)
            auto da = [&](int kt, uint32_t(&a)[4]) {
                const uint4 v = sm.D[warp][kt][lane];
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
            };
            uint32_t dnext[8][4];
            if (chain && l >= 1) {
                const int j0 = l == 5 ? jT_L5 : (l == 4 ? jT_L4H : (l == 3 ? jT_L3 : (l == 2 ? jT_L2 : jT_L1)));
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    float acc[8][4];
                    zero8(acc);
                    tring_gemm(acc, j0 + half * 8, 8, da, sm, rf, lane);
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) {
                        const int kt = half * 4 + nt / 2, rr = (nt & 1) * 2;
                        // ReLU mask of a_{l-1} (own rows) from the bits taken when it was staged
                        const uint32_t mb = ((half == 0 ? relu_lo : relu_hi) >> (8 * (nt / 2) + 2 * rr)) & 0xfu;
                        dnext[kt][rr] = pack_h2(mb & 1u ? acc[nt][0] : 0.f, mb & 2u ? acc[nt][1] : 0.f);
                        dnext[kt][rr + 1] = pack_h2(mb & 4u ? acc[nt][2] : 0.f, mb & 8u ? acc[nt][3] : 0.f);
                    }
                }
            }
            if (chain && has_in) {
                const int j0 = l == 4 ? jT_L4C : jT_L0C;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    float acc[8][4];
                    zero8(acc);
                    tring_gemm(acc, j0 + half * 8, 8, da, sm, rf, lane);
                    if constexpr (PER_SAMPLE) {
                        // this lane owns columns col, col+1 of rows g / g+8 for layers 4 and 0 alike: plain +=, no atomics
                        if (K.d_sample_warp_codes) {
                            const int64_t sa = row0 + g, sb = row0 + g + 8;
#pragma unroll
                            for (int nt = 0; nt < 8; ++nt) {
                                const int col = half * 64 + nt * 8 + 2 * q;
                                if (sa < n) {
                                    float2 *p = reinterpret_cast<float2 *>(K.d_sample_warp_codes + (size_t)sa * NSB_WARP_CODE_DIM + col);
                                    const float2 v = *p;
                                    *p = make_float2(v.x + acc[nt][0] * inv_ls, v.y + acc[nt][1] * inv_ls);
                                }
                                if (sb < n) {
                                    float2 *p = reinterpret_cast<float2 *>(K.d_sample_warp_codes + (size_t)sb * NSB_WARP_CODE_DIM + col);
                                    const float2 v = *p;
                                    *p = make_float2(v.x + acc[nt][2] * inv_ls, v.y + acc[nt][3] * inv_ls);
                                }
                            }
                        }
                    } else if (K.B.d_warp_codes) {
#pragma unroll
                        for (int nt = 0; nt < 8; ++nt) {
                            const int col = half * 64 + nt * 8 + 2 * q;
                            if (ts_uniform) {
                                float s0 = acc[nt][0] + acc[nt][2], s1 = acc[nt][1] + acc[nt][3];
#pragma unroll
                                for (int o = 4; o < 32; o <<= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
                                if (g == 0) {
                                    float *cp = K.B.d_warp_codes + (size_t)tsr[0] * NSB_WARP_CODE_DIM + col;
                                    if (s0 != 0.f) atomicAdd(cp, s0 * inv_ls);
                                    if (s1 != 0.f) atomicAdd(cp + 1, s1 * inv_ls);
                                }
                            } else {
                                float *cp0 = K.B.d_warp_codes + (size_t)tsr[0] * NSB_WARP_CODE_DIM + col;
                                float *cp1 = K.B.d_warp_codes + (size_t)tsr[1] * NSB_WARP_CODE_DIM + col;
                                if (acc[nt][0] != 0.f) atomicAdd(cp0, acc[nt][0] * inv_ls);
                                if (acc[nt][1] != 0.f) atomicAdd(cp0 + 1, acc[nt][1] * inv_ls);
                                if (acc[nt][2] != 0.f) atomicAdd(cp1, acc[nt][2] * inv_ls);
                                if (acc[nt][3] != 0.f) atomicAdd(cp1 + 1, acc[nt][3] * inv_ls);
                            }
                        }
                    }
                }
            }
            __syncthreads();   // D / X are rewritten by the next layer
            if (chain && l >= 1) {
#pragma unroll
                for (int kt = 0; kt < 8; ++kt)
#pragma unroll
                    for (int k = 0; k < 4; ++k) dcur[kt][k] = dnext[kt][k];
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < 6 * 128; i += kDbThreads) {
        const float v = (&sm.bias_acc[0][0])[i];
        if (v != 0.f) atomicAdd(K.B.d_stem_b + i, v * inv_ls);
    }
}

static int g_db_sms = 0;

}  // namespace nsb

using namespace nsb;

extern "C" size_t nsb_deform_packed_t_bytes(void) { return (size_t)kTSlabs * kDSlab; }

static int db_sms() {
    if (g_db_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_db_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_db_sms <= 0) g_db_sms = 132;
    }
    return g_db_sms;
}

extern "C" size_t nsb_deform_bwd_workspace_bytes(void) { return (size_t)db_sms() * kScrF4 * sizeof(float4); }

template <bool PER_SAMPLE>
static int launch_deform_bwd(const DeformBwdKArgsPS &K, int n_ctas, size_t smem, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(deform_bwd_kernel<PER_SAMPLE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(deform_bwd_kernel): %s", cudaGetErrorString(e)); return 1; }
        configured = true;
    }
    deform_bwd_kernel<PER_SAMPLE><<<n_ctas, kDbThreads, smem, st>>>(static_cast<const DeformBwdKArgsT<PER_SAMPLE> &>(K));
    return check_launch("deform_bwd_kernel");
}

extern "C" int nsb_deform_backward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                   const nsb_deform_bwd_args *args, void *stream) {
    if (!params || !opts || !samples || !args) { set_error("nsb_deform_backward: null argument"); return 1; }
    if (samples->n_samples <= 0) return 0;
    const bool per_sample = args->sample_warp_codes != nullptr;
    if (!args->deform_packed_t || !args->deform_acts || !args->deform_enc || !args->d_xs || !params->deform_packed_tb ||
        !params->deform_bias || (!params->warp_codes && !per_sample) || !(args->loss_scale > 0.f) || !args->d_stem_b ||
        !args->d_r_w || !args->d_r_b || !args->d_v_w || !args->d_v_b) {
        set_error("nsb_deform_backward: missing tensors");
        return 1;
    }
    for (int l = 0; l < 6; ++l)
        if (!args->d_stem_w[l]) { set_error("nsb_deform_backward: d_stem_w[%d] missing", l); return 1; }
    if (samples->sample_code_bias && !per_sample) {
        set_error("nsb_deform_backward: a per-sample code bias needs the per-sample warp codes (sample_warp_codes)");
        return 1;
    }
    if (!args->dw_workspace) { set_error("nsb_deform_backward: dw_workspace missing (nsb_deform_bwd_workspace_bytes)"); return 1; }
    db_sms();
    DeformBwdKArgsPS K;
    K.P = *params; K.O = *opts; K.S = *samples;
    std::memcpy(&K.B, args, sizeof(DeformBwdCore));
    for (int k = 0; k < 3; ++k) K.aabb_size[k] = params->aabb[3 + k] - params->aabb[k];
    K.sample_warp_codes = reinterpret_cast<const __half *>(args->sample_warp_codes);
    K.d_sample_warp_codes = args->d_sample_warp_codes;
    const size_t smem = sizeof(SmemDB);
    const int64_t n_tiles = (samples->n_samples + NSB_TILE - 1) / NSB_TILE;
    const int n_ctas = (int)std::min<int64_t>(n_tiles, g_db_sms);
    int rc = per_sample ? launch_deform_bwd<true>(K, n_ctas, smem, (cudaStream_t)stream)
                        : launch_deform_bwd<false>(K, n_ctas, smem, (cudaStream_t)stream);
    if (rc) return rc;
    DwReduceArgs R;
    R.scratch = reinterpret_cast<const float4 *>(args->dw_workspace);
    R.n_ctas = n_ctas;
    R.inv_ls = 1.0f / args->loss_scale;
    for (int l = 0; l < 6; ++l) R.d_stem_w[l] = args->d_stem_w[l];
    deform_dw_reduce_kernel<<<(kScrF4 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(R);
    return check_launch("deform_dw_reduce_kernel");
}
