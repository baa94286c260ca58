// Backward of the density/colour MLPs and of the hash ensemble (training), sm_90a.
//
// Replaces the autograd of (reference, relative to /root/reference/src/nersemble/nerfstudio/):
//   fields/nersemble_nerfacto_field.py:285-293,377   tcnn mlp_base / mlp_head backward, trunc_exp backward
//   field_components/hash_ensemble.py:102-156        einsum blend backward (-> time-code gradient)
//   tcnn kernel_grid_backward [3P]                   scatter of dL/dfeat into the hash tables
//
// field_mlp_bwd_kernel: 8 warps x 16 rows per 128-sample tile, everything in registers:
//   * forward activations are recomputed from the saved blended features (80 HMMA per 16 rows);
//   * deltas flow backwards through mma.sync with TRANSPOSED weight fragments (pack_field_bwd); the
//     accumulator layout of a delta tile is again the A-fragment layout of the next GEMM;
//   * weight gradients dW = delta^T . a are mma.sync too: both operands are transposed 8x8-blockwise with
//     movmatrix, accumulated into a per-CTA fp32 shared-memory copy, flushed once with global atomics.
//   Deltas are fp16 MMA operands -> a loss scale keeps them in range (tcnn does the same, x128).
// hash_bwd_kernel: one warp per sample, lane (g,q) = (corner, 8-member group) exactly like the forward
//   gather; per level one 32-byte load (values, for the time-code gradient) and four 16-byte vector reductions
//   (red.global.add.v4.f32) into the fp32 gradient line of the table entry.
#include <algorithm>
#include <cstddef>
#include <cstring>
#include <type_traits>

#include "nsb_common.cuh"
#include "nsb_gather.cuh"
#include "nsb_mlp.cuh"

namespace nsb {

// nsb_field_bwd_args without its trailing per-sample-code field.  The kernels of the training step take this as their
// parameter block, so the per-sample-code field appended to the C struct moves none of their parameter offsets (the
// second parameter of hash_expand_kernel would otherwise shift).
struct FieldBwdCore {
    const void *field_packed_t, *feat;
    const float *xs, *sigma, *rgb, *d_sigma, *d_rgb;
    float loss_scale;
    float *d_feat, *d_base_w, *d_head_w, *d_tables, *d_blend_codes, *d_xs, *g_rank1;
    const int32_t *ts_slot;
    int32_t n_slots;
    const void *corner_vals;
    float *cw_slots_out;
};
static_assert(sizeof(FieldBwdCore) == offsetof(nsb_field_bwd_args, d_sample_blend_codes) &&
              offsetof(FieldBwdCore, loss_scale) == offsetof(nsb_field_bwd_args, loss_scale) &&
              offsetof(FieldBwdCore, n_slots) == offsetof(nsb_field_bwd_args, n_slots) &&
              offsetof(FieldBwdCore, cw_slots_out) == offsetof(nsb_field_bwd_args, cw_slots_out),
              "FieldBwdCore must be the leading part of nsb_field_bwd_args");

struct FieldBwdKArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    FieldBwdCore B;
};

// hash_bwd_kernel modes: blend codes of the time-embedding table (training; the code gradient is summed per timestep),
// per-sample blend codes (component field: per-sample code gradient), and the stand-alone HashEnsemble (positions are
// the normalised hash input itself, S.positions [n][3], always in the box; d_feat is the output gradient).
enum HashBwdMode { kTableCodes = 0, kSampleCodes = 1, kBlendOnly = 2 };
struct FieldBwdKArgsPS : FieldBwdKArgs {
    float *d_sample_codes;   // [n][32] or NULL
};
template <int MODE>
using HashBwdKArgs = std::conditional_t<MODE == kTableCodes, FieldBwdKArgs, FieldBwdKArgsPS>;

constexpr int kBaseW = 64 * 32 + 16 * 64;             // 3072
constexpr int kHeadW = 64 * 32 + 64 * 64 + 16 * 64;   // 7168

// Weight gradients dW_l = delta_l^T . x_l are reduced over ALL 128 rows of the tile on the tensor cores: every warp
// stages its delta / input fragments (A-fragment order) in shared memory, then each warp owns 5 of the 40 16x16 output
// blocks, contracts over the 8 row blocks (movmatrix transposes, K = 128) and adds the result to its private slots of
// the per-CTA accumulator, which is kept in FRAGMENT order (conflict-free float4 per lane, no atomics).
// (First version: every warp formed the K = 16 product of its own rows and atomicAdd'ed it to a shared [out][in]
//  array: fp32 shared atomics are CAS loops -- ATOMS.CAST.SPIN, 8-way bank conflicts, 80 % of the kernel's samples.)
constexpr int kStD = 14, kStX = 16, kDwBlocks = 40;
struct DwBlock { uint8_t d, x, ob, ib, it; uint16_t base; };   // staged delta / input index, block coords, IT, flat offset
__constant__ DwBlock kDwBlk[kDwBlocks];

struct alignas(16) SmemBwd {
    uint4 wf[kFieldPackedU4];   // forward fragments
    uint4 wb[kFieldPackedU4];   // transposed fragments (dX GEMMs)
    float4 acc[kDwBlocks][2][32];   // per-CTA weight-gradient accumulator, fragment order [block][n-half][lane]
    union {
        struct { uint4 D[8][kStD][32]; uint4 X[8][kStX][32]; } st;   // per-tile staging
        float dw[kBaseW + kHeadW];                                      // flush: flat [out][in(kernel col order)]
    } u;
};

__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t a) {
    uint32_t d;
    asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
    return d;
}

// 32-bit mask of (acc > 0) in accumulator order [nt][4]
template <int NT>
__device__ __forceinline__ uint32_t relu_mask(const float (&acc)[NT][4]) {
    uint32_t m = 0;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) m |= (acc[nt][k] > 0.f ? 1u : 0u) << (nt * 4 + k);
    return m;
}

// delta (accumulator layout) -> masked -> A fragments of the next GEMM
template <int NT>
__device__ __forceinline__ void mask_pack(const float (&acc)[NT][4], uint32_t mask, uint32_t (&out)[NT / 2][4]) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float v0 = (mask >> (nt * 4 + 0)) & 1 ? acc[nt][0] : 0.f, v1 = (mask >> (nt * 4 + 1)) & 1 ? acc[nt][1] : 0.f;
        const float v2 = (mask >> (nt * 4 + 2)) & 1 ? acc[nt][2] : 0.f, v3 = (mask >> (nt * 4 + 3)) & 1 ? acc[nt][3] : 0.f;
        out[nt / 2][(nt & 1) * 2 + 0] = pack_h2(v0, v1);
        out[nt / 2][(nt & 1) * 2 + 1] = pack_h2(v2, v3);
    }
}

// park this warp's delta (OT k-tiles of 16 outputs) and layer-input (IT k-tiles) fragments for the tile-wide dW pass
template <int OT, int IT>
__device__ __forceinline__ void stage_dw(SmemBwd &sm, int warp, int d0, int x0, const uint32_t (&dA)[OT][4],
                                         const uint32_t (&xA)[IT][4], int lane) {
#pragma unroll
    for (int ob = 0; ob < OT; ++ob) sm.u.st.D[warp][d0 + ob][lane] = make_uint4(dA[ob][0], dA[ob][1], dA[ob][2], dA[ob][3]);
#pragma unroll
    for (int ib = 0; ib < IT; ++ib) sm.u.st.X[warp][x0 + ib][lane] = make_uint4(xA[ib][0], xA[ib][1], xA[ib][2], xA[ib][3]);
}

__global__ void __launch_bounds__(256, 1) field_mlp_bwd_kernel(const __grid_constant__ FieldBwdKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemBwd &sm = *reinterpret_cast<SmemBwd *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    const int64_t n = K.S.n_samples;
    const int64_t n_tiles = (n + NSB_TILE - 1) / NSB_TILE;
    {
        const uint4 *f = reinterpret_cast<const uint4 *>(K.P.field_packed);
        const uint4 *b = reinterpret_cast<const uint4 *>(K.B.field_packed_t);
        for (int i = tid; i < kFieldPackedU4; i += 256) { sm.wf[i] = __ldg(f + i); sm.wb[i] = __ldg(b + i); }
        for (int i = tid; i < kDwBlocks * 2 * 32; i += 256) (&sm.acc[0][0][0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    const float ls = K.B.loss_scale, inv_ls = 1.0f / K.B.loss_scale;
    const __half *featp = reinterpret_cast<const __half *>(K.B.feat);
    // weight-gradient slices inside sm.dw (kernel column order, flat [out][in])

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * NSB_TILE + warp * 16;   // (a warp whose rows are all >= n runs with zero deltas: barriers below)
        const int64_t ra = row0 + g, rb = row0 + g + 8;
        const bool va = ra < n, vb = rb < n;
        const int64_t sa = va ? ra : n - 1, sb = vb ? rb : n - 1;
        // ---------------- forward recompute ----------------
        uint32_t fa[2][4];
#pragma unroll
        for (int kt = 0; kt < 2; ++kt) {
            fa[kt][0] = __ldg(reinterpret_cast<const uint32_t *>(featp + sa * 32 + kt * 16 + 2 * q));
            fa[kt][1] = __ldg(reinterpret_cast<const uint32_t *>(featp + sb * 32 + kt * 16 + 2 * q));
            fa[kt][2] = __ldg(reinterpret_cast<const uint32_t *>(featp + sa * 32 + kt * 16 + 2 * q + 8));
            fa[kt][3] = __ldg(reinterpret_cast<const uint32_t *>(featp + sb * 32 + kt * 16 + 2 * q + 8));
        }
        float acc8[8][4];
        smem_gemm<2, 4>(acc8, fa, sm.wf, lane);
        const uint32_t m_b0 = relu_mask<8>(acc8);
        uint32_t h1[4][4];
        relu_pack_nobias<8>(acc8, h1);
        float b1acc[2][4];
        smem_gemm<4, 1>(b1acc, h1, sm.wf + 256, lane);
        // directions of the two rows
        float da[3] = {1.f, 1.f, 1.f}, db[3] = {1.f, 1.f, 1.f};
        if (K.S.origins != nullptr) {
            const int ria = K.S.ray_indices[sa], rib = K.S.ray_indices[sb];
#pragma unroll
            for (int k = 0; k < 3; ++k) { da[k] = K.S.directions[3 * (int64_t)ria + k]; db[k] = K.S.directions[3 * (int64_t)rib + k]; }
        } else if (K.S.sample_directions) {
#pragma unroll
            for (int k = 0; k < 3; ++k) { da[k] = K.S.sample_directions[3 * sa + k]; db[k] = K.S.sample_directions[3 * sb + k]; }
        }
        uint32_t ha[2][4];
        {
            float g00 = b1acc[0][0], g02 = b1acc[0][2];
            if (q == 0) { g00 = 1.0f; g02 = 1.0f; }
            ha[0][0] = pack_h2(g00, b1acc[0][1]);
            ha[0][1] = pack_h2(g02, b1acc[0][3]);
            ha[0][2] = pack_h2(b1acc[1][0], b1acc[1][1]);
            ha[0][3] = pack_h2(b1acc[1][2], b1acc[1][3]);
            const float ea0 = q == 0 ? (da[0] + 1.f) / 2.f : (q == 1 ? (da[2] + 1.f) / 2.f : 1.f), ea1 = q == 0 ? (da[1] + 1.f) / 2.f : 1.f;
            const float eb0 = q == 0 ? (db[0] + 1.f) / 2.f : (q == 1 ? (db[2] + 1.f) / 2.f : 1.f), eb1 = q == 0 ? (db[1] + 1.f) / 2.f : 1.f;
            ha[1][0] = pack_h2(ea0, ea1);
            ha[1][1] = pack_h2(eb0, eb1);
            ha[1][2] = pack_h2(1.0f, 1.0f);
            ha[1][3] = pack_h2(1.0f, 1.0f);
        }
        smem_gemm<2, 4>(acc8, ha, sm.wf + 384, lane);
        const uint32_t m_c0 = relu_mask<8>(acc8);
        uint32_t c1in[4][4];
        relu_pack_nobias<8>(acc8, c1in);
        smem_gemm<4, 4>(acc8, c1in, sm.wf + 640, lane);
        const uint32_t m_c1 = relu_mask<8>(acc8);
        uint32_t c2in[4][4];
        relu_pack_nobias<8>(acc8, c2in);
        // (the colour pre-activation itself is not needed: sigmoid' comes from the saved rgb)

        // ---------------- deltas ----------------
        // output delta: d rgb * rgb (1 - rgb) on columns 0..2 (lane q==0: cols 0,1; q==1: col 2)
        float dout[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        if (K.B.d_rgb && q < 2) {
            const int c0 = 2 * q;
            if (va) {
                const float r0 = K.B.rgb[3 * ra + c0];
                dout[0][0] = ls * K.B.d_rgb[3 * ra + c0] * r0 * (1.f - r0);
                if (q == 0) { const float r1 = K.B.rgb[3 * ra + 1]; dout[0][1] = ls * K.B.d_rgb[3 * ra + 1] * r1 * (1.f - r1); }
            }
            if (vb) {
                const float r0 = K.B.rgb[3 * rb + c0];
                dout[0][2] = ls * K.B.d_rgb[3 * rb + c0] * r0 * (1.f - r0);
                if (q == 0) { const float r1 = K.B.rgb[3 * rb + 1]; dout[0][3] = ls * K.B.d_rgb[3 * rb + 1] * r1 * (1.f - r1); }
            }
        }
        uint32_t dA1[1][4];
        mask_pack<2>(dout, 0xffu, dA1);
        stage_dw<1, 4>(sm, warp, 0, 0, dA1, c2in, lane);
        smem_gemm<1, 4>(acc8, dA1, sm.wb + 1152, lane);          // d c2in  [16 x 64]
        uint32_t dA4[4][4];
        mask_pack<8>(acc8, m_c1, dA4);
        stage_dw<4, 4>(sm, warp, 1, 4, dA4, c1in, lane);
        smem_gemm<4, 4>(acc8, dA4, sm.wb + 640, lane);           // d c1in  [16 x 64]
        mask_pack<8>(acc8, m_c0, dA4);
        stage_dw<4, 2>(sm, warp, 5, 8, dA4, ha, lane);
        float dh[4][4];
        smem_gemm<4, 2>(dh, dA4, sm.wb + 384, lane);             // d head input [16 x 32]; cols 1..15 = geo features
        // delta of the density-MLP output: col 0 = d sigma * exp(clamp(h0,-15,15)) * selector (trunc_exp backward)
        float dhb[2][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { dhb[0][k] = dh[0][k]; dhb[1][k] = dh[1][k]; }
        if (q == 0) {
            const float sela = va ? K.B.xs[4 * ra + 3] : 0.f, selb = vb ? K.B.xs[4 * rb + 3] : 0.f;
            const float dsa = (va && K.B.d_sigma) ? K.B.d_sigma[ra] : 0.f, dsb = (vb && K.B.d_sigma) ? K.B.d_sigma[rb] : 0.f;
            dhb[0][0] = ls * dsa * expf(fminf(fmaxf(b1acc[0][0], -15.f), 15.f)) * sela;
            dhb[0][2] = ls * dsb * expf(fminf(fmaxf(b1acc[0][2], -15.f), 15.f)) * selb;
        }
        mask_pack<2>(dhb, 0xffu, dA1);
        stage_dw<1, 4>(sm, warp, 9, 10, dA1, h1, lane);
        smem_gemm<1, 4>(acc8, dA1, sm.wb + 256, lane);           // d h1 [16 x 64]
        mask_pack<8>(acc8, m_b0, dA4);
        stage_dw<4, 2>(sm, warp, 10, 14, dA4, fa, lane);
        float dfe[4][4];
        smem_gemm<4, 2>(dfe, dA4, sm.wb, lane);                  // d feat [16 x 32]
        if (K.B.d_feat) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                if (va) *reinterpret_cast<float2 *>(K.B.d_feat + ra * 32 + nt * 8 + 2 * q) = make_float2(dfe[nt][0] * inv_ls, dfe[nt][1] * inv_ls);
                if (vb) *reinterpret_cast<float2 *>(K.B.d_feat + rb * 32 + nt * 8 + 2 * q) = make_float2(dfe[nt][2] * inv_ls, dfe[nt][3] * inv_ls);
            }
        }
        // ---------------- weight gradients: tile-wide contraction, 5 output blocks per warp ----------------
        __syncthreads();
#pragma unroll 1
        for (int bi = 0; bi < kDwBlocks / 8; ++bi) {
            const int blk = warp * (kDwBlocks / 8) + bi;
            const int di = kDwBlk[blk].d, xi = kDwBlk[blk].x;
            float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
            for (int r = 0; r < 8; ++r) {
                const uint4 d = sm.u.st.D[r][di][lane];
                const uint4 x = sm.u.st.X[r][xi][lane];
                // A = delta^T block [o 16][rows 16]: (o-lo,r-lo)=T(d0) (o-hi,r-lo)=T(d2) (o-lo,r-hi)=T(d1) (o-hi,r-hi)=T(d3)
                const uint32_t a[4] = {movmatrix_trans(d.x), movmatrix_trans(d.z), movmatrix_trans(d.y), movmatrix_trans(d.w)};
                mma16816(c0, a, movmatrix_trans(x.x), movmatrix_trans(x.y));   // input columns ib*16 + 0..7
                mma16816(c1, a, movmatrix_trans(x.z), movmatrix_trans(x.w));   // input columns ib*16 + 8..15
            }
            float4 v0 = sm.acc[blk][0][lane], v1 = sm.acc[blk][1][lane];
            v0.x += c0[0]; v0.y += c0[1]; v0.z += c0[2]; v0.w += c0[3];
            v1.x += c1[0]; v1.y += c1[1]; v1.z += c1[2]; v1.w += c1[3];
            sm.acc[blk][0][lane] = v0; sm.acc[blk][1][lane] = v1;
        }
        __syncthreads();   // staging is rewritten by the next tile
    }
    // fragment order -> flat [out][in(kernel col order)] (aliases the staging area)
    for (int i = tid; i < kDwBlocks * 2 * 32; i += 256) {
        const int l = i & 31, hn = (i >> 5) & 1, blk = i >> 6;
        const DwBlock b = kDwBlk[blk];
        const float4 v = sm.acc[blk][hn][l];
        const int o = b.ob * 16 + (l >> 2), c = b.ib * 16 + hn * 8 + 2 * (l & 3), ld = 16 * b.it;
        float *dst = sm.u.dw + b.base;
        dst[o * ld + c] = v.x; dst[o * ld + c + 1] = v.y; dst[(o + 8) * ld + c] = v.z; dst[(o + 8) * ld + c + 1] = v.w;
    }
    __syncthreads();
    // flush: kernel column order -> tcnn flat layout.  Only head layer 0 has permuted input columns:
    // kernel col k' -> reference col: 0 -> 18, 1..15 -> k'+2, 16..18 -> k'-16, 19..31 -> k'
    for (int i = tid; i < kBaseW + kHeadW; i += 256) {
        const float v = sm.u.dw[i] * inv_ls;
        if (v == 0.f) continue;
        if (i < kBaseW) {
            if (K.B.d_base_w) atomicAdd(K.B.d_base_w + i, v);
        } else if (K.B.d_head_w) {
            int j = i - kBaseW;
            if (j < 2048) {
                const int o = j >> 5, kp = j & 31;
                const int ref = kp == 0 ? 18 : (kp < 16 ? kp + 2 : (kp < 19 ? kp - 16 : kp));
                j = o * 32 + ref;
            }
            atomicAdd(K.B.d_head_w + j, v);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// table + time-code gradients: one warp per sample
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void red_add_v2(float *p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(256) hash_bwd_kernel(const __grid_constant__ HashBwdKArgs<MODE> K) {
    constexpr bool kPerSample = MODE != kTableCodes;
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const uint32_t dx = g & 1, dy = (g >> 1) & 1, dz = g >> 2;
    const int64_t n = K.S.n_samples;
    const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    // contiguous chunk of samples per warp: consecutive samples share a ray (same time code) and table lines
    const int64_t per = (n + n_warps - 1) / n_warps;
    const int64_t s_begin = warp_global * per, s_end = min(n, s_begin + per);
    const uint8_t *tab = reinterpret_cast<const uint8_t *>(K.P.tables) + q * 32;
    float code_acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int acc_ts = -1;
    auto flush_codes = [&]() {
        if (acc_ts >= 0 && K.B.d_blend_codes && g == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v = code_acc[j] * K.O.cw_scale[8 * q + j];     // cw = code*scale + bias
                if (v != 0.f) atomicAdd(K.B.d_blend_codes + (size_t)acc_ts * NSB_MEMBERS + 8 * q + j, v);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) code_acc[j] = 0.f;
    };
    for (int64_t s = s_begin; s < s_end; ++s) {
        float4 xs;
        if constexpr (MODE == kBlendOnly)
            xs = make_float4(K.S.positions[3 * s + 0], K.S.positions[3 * s + 1], K.S.positions[3 * s + 2], 1.0f);
        else
            xs = __ldg(reinterpret_cast<const float4 *>(K.B.xs) + s);
        bool rank1 = false;
        float *gslot = nullptr;
        const float *code_row;
        if constexpr (kPerSample) {
            code_row = K.S.sample_blend_codes + s * NSB_MEMBERS;
        } else {
            // timestep of the sample (same rounding as the forward)
            float tt = 0.f;
            if (K.S.origins != nullptr) { if (K.S.ray_times) tt = K.S.ray_times[K.S.ray_indices[s]]; }
            else if (K.S.sample_times) tt = K.S.sample_times[s];
            int ts = __float2int_rn(__fmul_rn(tt, (float)(K.P.n_timesteps - 1)));
            ts = min(max(ts, 0), K.P.n_timesteps - 1);
            if (ts != acc_ts) { flush_codes(); acc_ts = ts; }
            rank1 = K.B.g_rank1 != nullptr;
            if (rank1) {
                const int slot = K.B.ts_slot[ts];
                gslot = K.B.g_rank1 + (size_t)slot * ((size_t)K.P.levels.offset[NSB_MAX_LEVELS - 1] + K.P.levels.entries[NSB_MAX_LEVELS - 1]) * 2;
            }
            code_row = K.S.sample_blend_codes ? K.S.sample_blend_codes + s * NSB_MEMBERS
                                              : K.P.blend_codes + (size_t)ts * NSB_MEMBERS;
        }
        const float4 c0 = __ldg(reinterpret_cast<const float4 *>(code_row) + 2 * q);
        const float4 c1 = __ldg(reinterpret_cast<const float4 *>(code_row) + 2 * q + 1);
        const float craw[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
        float cw[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            // the forward rounds the blend weight to fp16 (B operand of the member reduction)
            cw[j] = __half2float(__float2half_rn(fmaf(craw[j], K.O.cw_scale[8 * q + j], K.O.cw_bias[8 * q + j])));
        }
        float dcw[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float ex = 0.f, ey = 0.f, ez = 0.f;   // dL/dx partial sums (this lane's corner and members)
#pragma unroll 2
        for (int l = 0; l < NSB_MAX_LEVELS; ++l) {
            const float2 df = __ldg(reinterpret_cast<const float2 *>(K.B.d_feat + s * 32) + l);
            const float scale = K.P.levels.scale[l];
            const uint32_t res = K.P.levels.res[l], ent = K.P.levels.entries[l], off = K.P.levels.offset[l];
            const float px = fmaf(scale, xs.x, 0.5f), py = fmaf(scale, xs.y, 0.5f), pz = fmaf(scale, xs.z, 0.5f);
            const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
            const float fx = px - flx, fy = py - fly, fz = pz - flz;
            const uint32_t cx = (uint32_t)(int)flx + dx, cy = (uint32_t)(int)fly + dy, cz = (uint32_t)(int)flz + dz;
            const float wx = dx ? fx : 1.0f - fx, wy = dy ? fy : 1.0f - fy, wz = dz ? fz : 1.0f - fz;
            const float w = (wx * wy) * wz;
            uint32_t idx;
            if (K.P.levels.hashed[l]) {
                idx = (cx ^ (cy * kPrimeY) ^ (cz * kPrimeZ)) & (ent - 1);
            } else {
                idx = cx + cy * res + cz * res * res;
                idx = idx >= ent ? idx - ent : idx;
            }
            const size_t entry = (size_t)(off + idx);
            const float g0 = w * df.x, g1 = w * df.y;
            if (rank1) {   // 2-vector per (timestep, line); member expansion and code gradient happen in hash_expand_kernel
                if (q == 0 && (g0 != 0.f || g1 != 0.f)) red_add_v2(gslot + entry * 2, g0, g1);
            }
            bool want_values;
            if constexpr (kPerSample) want_values = K.d_sample_codes || K.B.d_xs;
            else want_values = (K.B.d_blend_codes && !rank1) || K.B.d_xs;
            if (want_values) {
                uint32_t v[8];
                ldg256(tab + entry * 128, v);
                float pb0 = 0.f, pb1 = 0.f;   // this lane's share of the member-blended corner value
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 f = unpack_h2(v[j]);
                    dcw[j] = fmaf(g0, f.x, fmaf(g1, f.y, dcw[j]));
                    pb0 = fmaf(cw[j], f.x, pb0);
                    pb1 = fmaf(cw[j], f.y, pb1);
                }
                // d w / d x_d = +-scale * (product of the other two factors)   (frac = scale*x + 0.5 - floor)
                const float t = scale * (df.x * pb0 + df.y * pb1);
                ex = fmaf(dx ? t : -t, wy * wz, ex);
                ey = fmaf(dy ? t : -t, wx * wz, ey);
                ez = fmaf(dz ? t : -t, wx * wy, ez);
            }
            if (!rank1 && K.B.d_tables && (g0 != 0.f || g1 != 0.f)) {
                float *gl = K.B.d_tables + entry * 64 + q * 16;     // fp32 gradient line: [member 32][feat 2]
                red_add_v4(gl + 0, g0 * cw[0], g1 * cw[0], g0 * cw[1], g1 * cw[1]);
                red_add_v4(gl + 4, g0 * cw[2], g1 * cw[2], g0 * cw[3], g1 * cw[3]);
                red_add_v4(gl + 8, g0 * cw[4], g1 * cw[4], g0 * cw[5], g1 * cw[5]);
                red_add_v4(gl + 12, g0 * cw[6], g1 * cw[6], g0 * cw[7], g1 * cw[7]);
            }
        }
        if (K.B.d_xs) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                ex += __shfl_xor_sync(0xffffffffu, ex, o);
                ey += __shfl_xor_sync(0xffffffffu, ey, o);
                ez += __shfl_xor_sync(0xffffffffu, ez, o);
            }
            if (lane == 0) {   // positions outside the box were zeroed (x * selector): no gradient
                K.B.d_xs[3 * s + 0] = ex * xs.w; K.B.d_xs[3 * s + 1] = ey * xs.w; K.B.d_xs[3 * s + 2] = ez * xs.w;
            }
        }
        if constexpr (kPerSample) {
            if (K.d_sample_codes) {
                float v[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {   // sum over the 8 corner lanes (lane bits 2..4); cw = code*scale + bias
                    v[j] = dcw[j];
                    v[j] += __shfl_xor_sync(0xffffffffu, v[j], 4);
                    v[j] += __shfl_xor_sync(0xffffffffu, v[j], 8);
                    v[j] += __shfl_xor_sync(0xffffffffu, v[j], 16);
                    v[j] *= K.O.cw_scale[8 * q + j];
                }
                if (g == 0) {
                    float4 *dst = reinterpret_cast<float4 *>(K.d_sample_codes + s * NSB_MEMBERS) + 2 * q;
                    dst[0] = make_float4(v[0], v[1], v[2], v[3]);
                    dst[1] = make_float4(v[4], v[5], v[6], v[7]);
                }
            }
        } else if (K.B.d_blend_codes && !rank1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {   // sum over the 8 corner lanes (lane bits 2..4)
                float v = dcw[j];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                code_acc[j] += v;
            }
        }
    }
    if constexpr (!kPerSample) flush_codes();
}

// ---------------------------------------------------------------------------------------------
// Rank-1 scatter with the corner values the training forward saved (nsb_field_out.corner_vals): no table reads.
// One warp per sample, FOUR rounds: in round U lane L owns (level 4U + (L >> 3), corner L & 7) -- 32 distinct pairs per
// round, every index / weight computed once (the kernel above repeats them in the 4 lanes of a quad).  Per pair:
//   table gradient   G[slot][line] += w * dfeat[level]          (red.v2)
//   position gradient dL/dx_d += +-scale * (dfeat . blended corner value) * (product of the other two weight factors)
// A warp walks a contiguous run of samples (consecutive samples of a ray), so at the coarse levels a lane meets the
// same line again and again: it keeps the running 2-vector in registers and issues the atomic only when the line
// (or the slot) changes -- levels 0..5 need 9x..1.5x fewer atomics (cell size / sample spacing).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) hash_bwd_cv_kernel(const __grid_constant__ FieldBwdKArgs K) {
    const int lane = threadIdx.x & 31;
    const uint32_t dx = lane & 1, dy = (lane >> 1) & 1, dz = (lane >> 2) & 1;
    const int lsub = lane >> 3;
    const int64_t n = K.S.n_samples;
    const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t per = (n + n_warps - 1) / n_warps;
    const int64_t s_begin = warp_global * per, s_end = min(n, s_begin + per);
    const size_t total = (size_t)K.P.levels.offset[NSB_MAX_LEVELS - 1] + K.P.levels.entries[NSB_MAX_LEVELS - 1];
    const __half2 *cv = reinterpret_cast<const __half2 *>(K.B.corner_vals);
    float scale[4];
    uint32_t res[4], ent[4], off[4], hashed[4];
#pragma unroll
    for (int U = 0; U < 4; ++U) {
        const int l = 4 * U + lsub;
        scale[U] = K.P.levels.scale[l]; res[U] = K.P.levels.res[l]; ent[U] = K.P.levels.entries[l];
        off[U] = K.P.levels.offset[l]; hashed[U] = K.P.levels.hashed[l];
    }
    float *run_ptr[4] = {nullptr, nullptr, nullptr, nullptr};   // pending (slot, line) of each round and its running sum
    float run0[4] = {0.f, 0.f, 0.f, 0.f}, run1[4] = {0.f, 0.f, 0.f, 0.f};
    for (int64_t s = s_begin; s < s_end; ++s) {
        const float4 xs = __ldg(reinterpret_cast<const float4 *>(K.B.xs) + s);
        float tt = 0.f;
        if (K.S.origins != nullptr) { if (K.S.ray_times) tt = K.S.ray_times[K.S.ray_indices[s]]; }
        else if (K.S.sample_times) tt = K.S.sample_times[s];
        int ts = __float2int_rn(__fmul_rn(tt, (float)(K.P.n_timesteps - 1)));
        ts = min(max(ts, 0), K.P.n_timesteps - 1);
        float *gslot = K.B.g_rank1 + (size_t)K.B.ts_slot[ts] * total * 2;
        float ex = 0.f, ey = 0.f, ez = 0.f;
#pragma unroll
        for (int U = 0; U < 4; ++U) {
            const float2 df = __ldg(reinterpret_cast<const float2 *>(K.B.d_feat + s * 32) + 4 * U + lsub);
            const float px = fmaf(scale[U], xs.x, 0.5f), py = fmaf(scale[U], xs.y, 0.5f), pz = fmaf(scale[U], xs.z, 0.5f);
            const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
            const float fx = px - flx, fy = py - fly, fz = pz - flz;
            const uint32_t cx = (uint32_t)(int)flx + dx, cy = (uint32_t)(int)fly + dy, cz = (uint32_t)(int)flz + dz;
            const float wx = dx ? fx : 1.0f - fx, wy = dy ? fy : 1.0f - fy, wz = dz ? fz : 1.0f - fz;
            const float w = (wx * wy) * wz;
            const uint32_t ih = (cx ^ (cy * kPrimeY) ^ (cz * kPrimeZ)) & (ent[U] - 1);
            uint32_t id = cx + cy * res[U] + cz * res[U] * res[U];
            id = id >= ent[U] ? id - ent[U] : id;
            float *dst = gslot + (size_t)(off[U] + (hashed[U] ? ih : id)) * 2;
            const float g0 = w * df.x, g1 = w * df.y;
            if (dst == run_ptr[U]) {
                run0[U] += g0; run1[U] += g1;
            } else {
                if (run_ptr[U] && (run0[U] != 0.f || run1[U] != 0.f)) red_add_v2(run_ptr[U], run0[U], run1[U]);
                run_ptr[U] = dst; run0[U] = g0; run1[U] = g1;
            }
            if (K.B.d_xs) {
                const float2 pb = __half22float2(cv[s * 128 + (4 * U + lsub) * 8 + (lane & 7)]);
                const float t = scale[U] * (df.x * pb.x + df.y * pb.y);   // frac = scale*x + 0.5 - floor
                ex = fmaf(dx ? t : -t, wy * wz, ex);
                ey = fmaf(dy ? t : -t, wx * wz, ey);
                ez = fmaf(dz ? t : -t, wx * wy, ez);
            }
        }
        if (K.B.d_xs) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                ex += __shfl_xor_sync(0xffffffffu, ex, o);
                ey += __shfl_xor_sync(0xffffffffu, ey, o);
                ez += __shfl_xor_sync(0xffffffffu, ez, o);
            }
            if (lane == 0) {   // positions outside the box were zeroed (x * selector): no gradient
                K.B.d_xs[3 * s + 0] = ex * xs.w; K.B.d_xs[3 * s + 1] = ey * xs.w; K.B.d_xs[3 * s + 2] = ez * xs.w;
            }
        }
    }
#pragma unroll
    for (int U = 0; U < 4; ++U)
        if (run_ptr[U] && (run0[U] != 0.f || run1[U] != 0.f)) red_add_v2(run_ptr[U], run0[U], run1[U]);
}

// ---------------------------------------------------------------------------------------------
// rank-1 expansion: d_tables[line][m][f] += sum_slots cw_slot[m] * G[slot][line][f];
//                   d_codes[t][m]       += scale[m] * sum_lines sum_f V[line][m][f] * G[slot(t)][line][f]
// one warp per table line (lane = member), grid-stride; G lines that were never touched are skipped.
// ---------------------------------------------------------------------------------------------
constexpr int kMaxSlots = 32;
constexpr int kExpWarps = 4, kExpLines = 32;

// Block form (same as table_step_kernel, nsb_optim.cu): a warp owns 32 consecutive lines per iteration, reads every
// slot's 2-vectors of those lines with one coalesced 256 B load per slot into a shared-memory panel, and then visits
// only the lines some slot touched (lane = member; the fp16 table line is one coalesced 128 B read, four lines in flight).
// TABLES = false (fused optimiser: the dense table gradient is never materialised): only the time-code gradient
// is computed -- the member expansion's two FMAs per (line, slot) are compiled out.
template <bool TABLES>
__global__ void __launch_bounds__(kExpWarps * 32) hash_expand_kernel(const __grid_constant__ FieldBwdKArgs K, size_t total_entries) {
    __shared__ float cw_s[kMaxSlots][NSB_MEMBERS];
    __shared__ int slot_ts[kMaxSlots];
    __shared__ float2 gs[kExpWarps][kMaxSlots][kExpLines];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_slots = K.B.n_slots;
    for (int i = threadIdx.x; i < kMaxSlots; i += blockDim.x) slot_ts[i] = -1;
    __syncthreads();
    for (int t = threadIdx.x; t < K.P.n_timesteps; t += blockDim.x) {
        const int sl = K.B.ts_slot[t];
        if (sl >= 0) slot_ts[sl] = t;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_slots * NSB_MEMBERS; i += blockDim.x) {
        const int sl = i / NSB_MEMBERS, m = i % NSB_MEMBERS, t = slot_ts[sl];
        float c = 0.f;
        if (t >= 0) c = __half2float(__float2half_rn(fmaf(K.P.blend_codes[(size_t)t * NSB_MEMBERS + m], K.O.cw_scale[m], K.O.cw_bias[m])));
        cw_s[sl][m] = c;
        if (K.B.cw_slots_out && blockIdx.x == 0) K.B.cw_slots_out[i] = c;
    }
    __syncthreads();
    if (!K.B.d_tables && !K.B.d_blend_codes) return;    // launched only to publish cw_slots_out
    float cw[kMaxSlots], dcode[kMaxSlots];
#pragma unroll
    for (int sl = 0; sl < kMaxSlots; ++sl) { dcode[sl] = 0.f; cw[sl] = sl < n_slots ? cw_s[sl][lane] : 0.f; }
    const __half2 *tab = reinterpret_cast<const __half2 *>(K.P.tables);
    const int64_t E = (int64_t)total_entries;
    const int64_t n_blocks = (E + kExpLines - 1) / kExpLines;
    for (int64_t blk = (int64_t)blockIdx.x * kExpWarps + warp; blk < n_blocks; blk += (int64_t)gridDim.x * kExpWarps) {
        const int64_t e0 = blk * kExpLines;
        {   // pull the NEXT block's workspace rows (n_slots x 256 B) and table lines (32 x 128 B) into L2
            const int64_t nb = blk + (int64_t)gridDim.x * kExpWarps;
            if (nb < n_blocks) {
                const int64_t ne = nb * kExpLines;
                for (int i = lane; i < 2 * n_slots; i += 32)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(K.B.g_rank1 + ((size_t)(i >> 1) * E + ne) * 2 + (i & 1) * 32));
                if (K.B.d_blend_codes && ne + lane < E)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(tab + (size_t)(ne + lane) * NSB_MEMBERS));
            }
        }
        unsigned any_slot = 0;
        bool mine = false;      // line e0 + lane touched in some slot
        for (int s0 = 0; s0 < n_slots; s0 += 8) {      // 8 slot rows in flight (a ballot per load serialises them)
            float2 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                v[u] = make_float2(0.f, 0.f);
                if (s0 + u < n_slots && e0 + lane < E)
                    v[u] = __ldg(reinterpret_cast<const float2 *>(K.B.g_rank1 + ((size_t)(s0 + u) * E + e0 + lane) * 2));
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (s0 + u >= n_slots) break;
                gs[warp][s0 + u][lane] = v[u];
                const bool nz = v[u].x != 0.f || v[u].y != 0.f;
                mine |= nz;
                if (__ballot_sync(0xffffffffu, nz)) any_slot |= 1u << (s0 + u);
            }
        }
        __syncwarp();
        unsigned todo = __ballot_sync(0xffffffffu, mine);
        while (todo) {
            int js[4];
            float2 vs[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {       // up to four touched lines in flight
                js[u] = todo ? __ffs(todo) - 1 : -1;
                if (todo) todo &= todo - 1;
                vs[u] = make_float2(0.f, 0.f);
                if (js[u] >= 0 && K.B.d_blend_codes) vs[u] = __half22float2(tab[(size_t)(e0 + js[u]) * NSB_MEMBERS + lane]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (js[u] < 0) continue;
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int sl = 0; sl < kMaxSlots; ++sl) {
                    if (!((any_slot >> sl) & 1)) continue;     // warp-uniform
                    const float2 gv = gs[warp][sl][js[u]];
                    if (TABLES) {
                        a0 = fmaf(cw[sl], gv.x, a0);
                        a1 = fmaf(cw[sl], gv.y, a1);
                    }
                    dcode[sl] = fmaf(vs[u].x, gv.x, fmaf(vs[u].y, gv.y, dcode[sl]));
                }
                if (TABLES && K.B.d_tables) {
                    float2 *dst = reinterpret_cast<float2 *>(K.B.d_tables + ((size_t)(e0 + js[u]) * NSB_MEMBERS + lane) * 2);
                    float2 cur = *dst;
                    cur.x += a0; cur.y += a1;
                    *dst = cur;
                }
            }
        }
        __syncwarp();
    }
    if (K.B.d_blend_codes) {
#pragma unroll
        for (int sl = 0; sl < kMaxSlots; ++sl) {
            const int t = sl < n_slots ? slot_ts[sl] : -1;
            if (t >= 0 && dcode[sl] != 0.f)
                atomicAdd(K.B.d_blend_codes + (size_t)t * NSB_MEMBERS + lane, dcode[sl] * K.O.cw_scale[lane]);
        }
    }
}

static int g_bwd_sms = 0;
static void bwd_sms() {
    if (g_bwd_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_bwd_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_bwd_sms <= 0) g_bwd_sms = 132;
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_field_backward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                  const nsb_field_bwd_args *args, void *stream) {
    if (!params || !opts || !samples || !args) { set_error("nsb_field_backward: null argument"); return 1; }
    if (samples->n_samples <= 0) return 0;
    if (!args->field_packed_t || !params->field_packed || !args->feat || !args->xs || !args->sigma ||
        (!args->rgb && args->d_rgb) || !args->d_feat || !(args->loss_scale > 0.f)) {
        set_error("nsb_field_backward: missing saved tensors / workspace / loss_scale");
        return 1;
    }
    const bool per_sample = args->d_sample_blend_codes != nullptr;
    const bool hash_pass = args->d_tables || args->d_blend_codes || args->d_xs || per_sample;
    if (hash_pass && (!params->tables || (!params->blend_codes && !samples->sample_blend_codes))) {
        set_error("nsb_field_backward: tables / blend codes missing");
        return 1;
    }
    if (per_sample && (!samples->sample_blend_codes || args->g_rank1)) {
        set_error("nsb_field_backward: d_sample_blend_codes needs per-sample blend codes and the direct scatter (no g_rank1)");
        return 1;
    }
    if (params->levels.n_levels != NSB_MAX_LEVELS) { set_error("nsb_field_backward: n_levels must be 16"); return 1; }
    bwd_sms();
    cudaStream_t st = (cudaStream_t)stream;
    FieldBwdKArgs K;
    K.P = *params; K.O = *opts; K.S = *samples;
    std::memcpy(&K.B, args, sizeof(FieldBwdCore));
    static bool configured = false;
    {   // 16x16 output blocks of the five weight matrices, in flat-accumulator order (see SmemBwd)
        static bool table_done_dev[64] = {};
        int dev = 0;
        cudaGetDevice(&dev);
        bool &table_done = table_done_dev[dev & 63];
        if (!table_done) {
            DwBlock t[kDwBlocks];
            int n = 0;
            struct { int d0, x0, OT, IT, base; } L[5] = {
                {0, 0, 1, 4, kBaseW + 2048 + 4096},   // head layer 2 (16 x 64)
                {1, 4, 4, 4, kBaseW + 2048},          // head layer 1 (64 x 64)
                {5, 8, 4, 2, kBaseW},                 // head layer 0 (64 x 32)
                {9, 10, 1, 4, 2048},                  // base layer 1 (16 x 64)
                {10, 14, 4, 2, 0}};                   // base layer 0 (64 x 32)
            for (auto &l : L)
                for (int ob = 0; ob < l.OT; ++ob)
                    for (int ib = 0; ib < l.IT; ++ib)
                        t[n++] = DwBlock{(uint8_t)(l.d0 + ob), (uint8_t)(l.x0 + ib), (uint8_t)ob, (uint8_t)ib, (uint8_t)l.IT, (uint16_t)l.base};
            cudaError_t e = cudaMemcpyToSymbol(kDwBlk, t, sizeof(t));
            if (e != cudaSuccess || n != kDwBlocks) { set_error("field_mlp_bwd: block table upload failed: %s", cudaGetErrorString(e)); return 1; }
            table_done = true;
        }
    }
    const size_t smem = sizeof(SmemBwd);
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(field_mlp_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(field_mlp_bwd_kernel): %s", cudaGetErrorString(e)); return 1; }
        configured = true;
    }
    const int64_t n_tiles = (samples->n_samples + NSB_TILE - 1) / NSB_TILE;
    field_mlp_bwd_kernel<<<(int)std::min<int64_t>(n_tiles, g_bwd_sms), 256, smem, st>>>(K);
    int rc = check_launch("field_mlp_bwd_kernel");
    if (rc) return rc;
    if (hash_pass) {
        const int blocks = (int)std::min<int64_t>((samples->n_samples + 7) / 8, (int64_t)g_bwd_sms * 8);
        if (per_sample) {
            FieldBwdKArgsPS KP;
            static_cast<FieldBwdKArgs &>(KP) = K;
            KP.d_sample_codes = args->d_sample_blend_codes;
            hash_bwd_kernel<kSampleCodes><<<blocks, 256, 0, st>>>(KP);
            return check_launch("hash_bwd_kernel");
        }
        if (args->g_rank1) {
            if (!args->ts_slot || args->n_slots < 1 || args->n_slots > kMaxSlots || samples->sample_blend_codes) {
                set_error("nsb_field_backward: rank-1 path needs ts_slot, 1 <= n_slots <= 32 and table-indexed blend codes");
                return 1;
            }
        }
        if (args->g_rank1 && args->corner_vals && !samples->sample_blend_codes) {
            hash_bwd_cv_kernel<<<blocks, 256, 0, st>>>(K);
            rc = check_launch("hash_bwd_cv_kernel");
        } else {
            hash_bwd_kernel<kTableCodes><<<blocks, 256, 0, st>>>(K);
            rc = check_launch("hash_bwd_kernel");
        }
        if (rc) return rc;
        if (args->g_rank1 && (args->d_tables || args->d_blend_codes || args->cw_slots_out)) {
            const size_t total = (size_t)params->levels.offset[NSB_MAX_LEVELS - 1] + params->levels.entries[NSB_MAX_LEVELS - 1];
            if (K.B.d_tables) hash_expand_kernel<true><<<g_bwd_sms * 6, kExpWarps * 32, 0, st>>>(K, total);
            else hash_expand_kernel<false><<<g_bwd_sms * 6, kExpWarps * 32, 0, st>>>(K, total);
            rc = check_launch("hash_expand_kernel");
        }
    }
    return rc;
}

extern "C" int nsb_hash_blend_backward(const nsb_field_params *params, const nsb_field_opts *opts, const float *x,
                                       const float *codes, int64_t n, const float *d_out, float *d_tables, float *d_codes,
                                       float *d_x, void *stream) {
    if (!params || !opts || !x || !codes || !d_out) { set_error("nsb_hash_blend_backward: null argument"); return 1; }
    if (n <= 0 || !(d_tables || d_codes || d_x)) return 0;
    if (!params->tables) { set_error("nsb_hash_blend_backward: tables missing"); return 1; }
    if (params->levels.n_levels != NSB_MAX_LEVELS) { set_error("nsb_hash_blend_backward: n_levels must be 16"); return 1; }
    bwd_sms();
    FieldBwdKArgsPS K = {};
    K.P = *params; K.O = *opts;
    K.S.n_samples = n;
    K.S.positions = x;
    K.S.sample_blend_codes = codes;
    K.B.d_feat = const_cast<float *>(d_out);     // read only
    K.B.d_tables = d_tables;
    K.B.d_xs = d_x;
    K.d_sample_codes = d_codes;
    const int blocks = (int)std::min<int64_t>((n + 7) / 8, (int64_t)g_bwd_sms * 8);
    hash_bwd_kernel<kBlendOnly><<<blocks, 256, 0, (cudaStream_t)stream>>>(K);
    return check_launch("hash_bwd_kernel");
}
