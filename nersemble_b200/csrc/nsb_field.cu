// Fused per-sample field evaluation for sm_90a:
//   windowed posenc + warp code -> SE(3) deformation MLP (tensor cores) -> warp ->
//   32-member hash-ensemble gather + time-latent blend (HBM-bound) -> density MLP -> colour MLP.
//
// Replaces (reference, relative to /root/reference/src/nersemble/nerfstudio/):
//   field_components/deformation_field.py:77-107,148-166   SE3WarpingField / compute_offsets
//   field_components/windowed_nerf_encoding.py:33-74       WindowedNeRFEncoding
//   field_components/hash_ensemble.py:93-158                HashEnsemble.forward (8 tcnn grids + einsum)
//   fields/nersemble_nerfacto_field.py:250-301,303-383      get_density / get_outputs (tcnn MLPs)
//
// Work decomposition: see the comment block above field_kernel_ws (persistent, one CTA per SM, warp-specialised:
// tensor warps run the deformation MLP and the density/colour MLPs on mma.sync with the deformation weights
// streamed through a cp.async.bulk ring; gather warps do nothing but the 128-byte-line hash gather).
#include <algorithm>
#include <cstdlib>
#include <cstring>

#define NSB_NO_SPIN_GUARD 1   // see nsb_common.cuh mbar_wait
#include "nsb_common.cuh"
#include "nsb_gather.cuh"
#include "nsb_march.cuh"
#include "nsb_mlp.cuh"
#include "nsb_tc.cuh"

namespace nsb {

constexpr int kSlabBytes = 2048;  // one k-tile (16) x 64 output columns, fragment order
constexpr int kChunkSlabs = 4;
constexpr int kChunkBytes = kSlabBytes * kChunkSlabs;
constexpr int kStages = 4;
constexpr int kBiasFloats = 6 * 128 + 8;

struct FieldArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    nsb_field_out out;
    float aabb_size[3];
};

__device__ __forceinline__ void zero_acc(float (&acc)[8][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;
}

// -------------------------------------------------------------------------------------------
// SE(3) exponential map applied to p (util/pytorch3d.py:107-191 + deformation_field.py:95-107)
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void cross3(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ void se3_apply(const float p[3], const float r[3], const float v[3], float out[3]) {
    float n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    float th = sqrtf(fmaxf(n2, 1e-4f));
    float s, c;
    sincosf(th, &s, &c);
    float f1 = s / th, f2 = (1.0f - c) / (th * th), f3 = (th - s) / (th * th * th);
    float rp[3], rrp[3], rv[3], rrv[3];
    cross3(r, p, rp); cross3(r, rp, rrp); cross3(r, v, rv); cross3(r, rv, rrv);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float o = (p[k] + f1 * rp[k] + f2 * rrp[k]) + (v[k] + f2 * rv[k] + f3 * rrv[k]);
        out[k] = isnan(o) ? p[k] : o;
    }
}

// ===========================================================================================
// v2: warp-specialised persistent kernel, 1 CTA per SM (with every warp doing every stage the gather is
// latency-bound on the number of gathering warps and cannot overlap the deformation phase).
//   8 TENSOR warps: deformation MLP of tile i+1 (16 rows each), then density+colour MLPs of tile i.  Tensor warp 0
//     lane 0 also refills the weight ring.
//   GATHER warps: nothing but the hash-ensemble gather; rows of a tile are claimed dynamically; each warp keeps
//     2 m-tiles (2 x 2 x 32 B per lane) in flight.
// Hand-off through shared memory, double-buffered by tile parity, two mbarrier arrays:
//   xs_full[b]   tensor -> gather : warped positions of tile i are in sm.xs[b]
//   feat_full[b] gather -> tensor : blended features of tile i are in sm.feat[b]
// The reverse (buffer-free) edges are implied by program order: tensor warps issue D(i+2) only after
// F(i), which waited for feat_full(i), i.e. for every gather warp to be done with tile i.
// ===========================================================================================
constexpr int kMT = 1;                            // m-tiles (16 rows) per tensor warp
constexpr int kTRows = 16 * kMT;                  // rows per tensor warp
constexpr int kTensorWarps = NSB_TILE / kTRows;   // 8
constexpr int kGatherWarps = 8;                   // multiple of 4: setmaxnreg works on warpgroups
constexpr int kThreadsWS = (kTensorWarps + kGatherWarps) * 32;
// Register budget: the kernels are launched with kLaunchRegs registers per thread (the SM's 65536 over the CTA's threads,
// in units of 8).  setmaxnreg can only move registers WITHIN the CTA's allocation (inc blocks until a dec released
// enough -- an inc that exceeds the pool hangs the kernel), so
//   kTensorWarps*32*kTensorRegs + kGatherWarps*32*kGatherRegs <= kThreadsWS*kLaunchRegs.
// 16 warps (128 registers at launch): the gather role gets 120 and the tensor role 136.  With more gather warps (and so
// fewer registers per thread) sm_90 ptxas spills in the gather role's sample loop, and the wgmma tensor role spills below
// 104 registers (tools/spill_report.py).
constexpr int kLaunchRegs = (65536 / kThreadsWS) & ~7;
constexpr int kGatherRegs = 120;
constexpr int kTensorRegs = 136;
static_assert(kTensorWarps * 32 * kTensorRegs + kGatherWarps * 32 * kGatherRegs <= kThreadsWS * kLaunchRegs, "register pool");
constexpr int kLaunchBoundWS = kThreadsWS;
// Slab layout of deform_packed_tb: layers 0 and 4 without their 128 warp-code columns (those enter as the
// per-timestep bias deform_code_bias[t][0|1][128]).
constexpr int kT_L0 = 0;                  // 2 x 3
constexpr int kT_L1 = kT_L0 + 6;          // 2 x 8
constexpr int kT_L2 = kT_L1 + 16;
constexpr int kT_L3 = kT_L2 + 16;
constexpr int kT_L4 = kT_L3 + 16;         // 2 x 11
constexpr int kT_L5 = kT_L4 + 22;         // 2 x 8
constexpr int kT_HEADS = kT_L5 + 16;      // 92
constexpr int kTbNumSlabs = kT_HEADS + 2; // 94
constexpr int kTbNumChunks = (kTbNumSlabs + kChunkSlabs - 1) / kChunkSlabs;  // 24
static_assert(kTbNumChunks % (2 * kStages) == 0 && kT_HEADS % kChunkSlabs == 0, "ring parity / heads chunk");
static_assert(kTensorWarps % 4 == 0 && kGatherWarps % 4 == 0, "setmaxnreg works on warpgroups");

struct alignas(16) TensorScratch {
    float pos[kTRows][4];          // world position xyz, w = timestep (int bits)
    float dirsel[2][kTRows][4];    // [tile parity] ray direction xyz, w = in-box selector
    uint4 enc[kMT][3][32];         // posenc A fragments [m-tile][k-tile][lane]
    uint4 act[2][kMT][8][32];      // [ping-pong][m-tile][k-tile][lane] hidden activations (lane-private)
};

struct alignas(128) SmemWS {
    uint8_t ring[kStages][kChunkBytes];
    uint4 field_w[kFieldPackedU4];
    float bias[kBiasFloats];
    uint64_t full[kStages];
    uint64_t empty[kStages];
    uint64_t xs_full[2];
    uint64_t feat_full[2];
    int tile_ctr[2];
    int64_t n_dyn;                          // fused render kernel: the packed sample count (known on the device only)
    uint64_t sampler_done;                  // fused render kernel: mbarrier, the tensor warps' sampler phase -> the gather warps
    alignas(16) float xs[2][NSB_TILE][4];  // normalised warped position (0 outside the box), w = timestep bits
    alignas(16) __half feat[2][NSB_TILE * kFeatStride];
    TensorScratch ts[kTensorWarps];
    uint2 blend_b[kGatherWarps][4 * 32];   // per gather warp: the current timestep's B fragments (lane-private columns)
    uint4 cv_stage[kGatherWarps][32];      // per gather warp: the current sample's corner values (training forward)
};

struct RingRefill {
    bool active;           // tensor warp 0, lane 0
    uint32_t gbase;        // global chunk index of this tile's chunk 0
    uint32_t total;        // chunks this CTA will consume in total
    const uint8_t *src;
    __device__ __forceinline__ void issue(SmemWS &sm, uint32_t gt) const {
        if (active && gt < total) {
            const uint32_t s = gt % kStages, kf = gt / kStages, c = gt % kTbNumChunks;
            mbar_wait<20>(&sm.empty[s], (kf & 1) ^ 1);   // every tensor warp released the previous use
            const uint32_t bytes = (c == kTbNumChunks - 1) ? (kTbNumSlabs - c * kChunkSlabs) * kSlabBytes : kChunkBytes;
            mbar_expect_tx(&sm.full[s], bytes);
            bulk_g2s(sm.ring[s], src + (size_t)c * kChunkBytes, bytes, &sm.full[s]);
        }
    }
};

// one N-half of a deformation layer for TWO m-tiles (32 rows): each B fragment pair feeds 4 HMMAs
template <class AFn>
__device__ __forceinline__ void ring_gemm2(float (&acc)[kMT][8][4], const int j0, const int KT, AFn &&afn, SmemWS &sm,
                                           const RingRefill &rf, int lane) {
    static_assert(kChunkSlabs == 4 && kStages == 4 && kTbNumChunks % (2 * kStages) == 0, "ring index arithmetic");
#pragma unroll 2
    for (int kt = 0; kt < KT; ++kt) {
        const int j = j0 + kt;
        const int chunk = j >> 2, stage = chunk & 3;
        if ((j & 3) == 0) {
            rf.issue(sm, rf.gbase + chunk + (kStages - 1));   // refill three chunks ahead
            __syncwarp();
            mbar_wait<20>(&sm.full[stage], (chunk >> 2) & 1);
        }
        uint32_t a[kMT][4];
#pragma unroll
        for (int m = 0; m < kMT; ++m) afn(m, kt, a[m]);
        const uint4 *slab = reinterpret_cast<const uint4 *>(&sm.ring[stage][(j & 3) * kSlabBytes]);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const uint4 b = slab[p * 32 + lane];
#pragma unroll
            for (int m = 0; m < kMT; ++m) {
                mma16816(acc[m][2 * p], a[m], b.x, b.y);
                mma16816(acc[m][2 * p + 1], a[m], b.z, b.w);
            }
        }
        if ((j & 3) == 3) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty[stage]);
        }
    }
}

// bias + ReLU + pack one N-half straight into the ping-pong activation buffer.
//   CODE = false: `sbias` is the layer's shared bias row (smem), one load serves both row halves.
//   CODE = true : layers 0 / 4 -- `gbias` is the per-timestep code-bias table (global, L1/L2 resident: 24 x 1 KB) and
//                 off[m][0|1] the float offset of the bias row of the m-tile's rows g / g+8.  Offsets instead of
//                 pointers: four 64-bit row pointers per m-tile cost 8 registers for the whole MLP.
template <int HALF, bool CODE>
__device__ __forceinline__ void relu_store2(const float (&acc)[kMT][8][4], uint4 (*dst)[8][32], const float *sbias,
                                            const float *gbias, const uint32_t (&off)[kMT][2], int q, int lane) {
#pragma unroll
    for (int m = 0; m < kMT; ++m) {
#pragma unroll
        for (int kt = 0; kt < 4; ++kt) {
            uint32_t r[4];
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const int nt = 2 * kt + o, col = HALF * 64 + nt * 8 + 2 * q;
                float2 b0, b1;
                if (CODE) {
                    b0 = __ldg(reinterpret_cast<const float2 *>(gbias + off[m][0] + col));
                    b1 = __ldg(reinterpret_cast<const float2 *>(gbias + off[m][1] + col));
                } else {
                    b0 = *reinterpret_cast<const float2 *>(sbias + col);
                    b1 = b0;
                }
                r[o * 2 + 0] = pack_h2(fmaxf(acc[m][nt][0] + b0.x, 0.f), fmaxf(acc[m][nt][1] + b0.y, 0.f));
                r[o * 2 + 1] = pack_h2(fmaxf(acc[m][nt][2] + b1.x, 0.f), fmaxf(acc[m][nt][3] + b1.y, 0.f));
            }
            dst[m][HALF * 4 + kt][lane] = make_uint4(r[0], r[1], r[2], r[3]);
        }
    }
}

__device__ __forceinline__ void zero_acc2(float (&acc)[kMT][8][4]) {
#pragma unroll
    for (int m = 0; m < kMT; ++m) zero_acc(acc[m]);
}

// density + colour MLPs for one m-tile (16 rows); feat rows / dirsel rows are this m-tile's row 0
template <bool HEAD>
__device__ __forceinline__ void field_mlp_tile(const FieldArgs &A, const uint4 *field_w, const __half *feat,
                                               const float (*dirsel)[4], int64_t row0, int64_t n, int lane) {
    const int g = lane >> 2, q = lane & 3;
    uint32_t fa[2][4];
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
        fa[kt][0] = *reinterpret_cast<const uint32_t *>(&feat[g * kFeatStride + kt * 16 + 2 * q]);
        fa[kt][1] = *reinterpret_cast<const uint32_t *>(&feat[(g + 8) * kFeatStride + kt * 16 + 2 * q]);
        fa[kt][2] = *reinterpret_cast<const uint32_t *>(&feat[g * kFeatStride + kt * 16 + 2 * q + 8]);
        fa[kt][3] = *reinterpret_cast<const uint32_t *>(&feat[(g + 8) * kFeatStride + kt * 16 + 2 * q + 8]);
    }
    float b0acc[8][4];
    smem_gemm<2, 4>(b0acc, fa, field_w, lane);
    uint32_t h1[4][4];
    relu_pack_nobias<8>(b0acc, h1);
    float b1acc[2][4];
    smem_gemm<4, 1>(b1acc, h1, field_w + 256, lane);
    const float sel0 = dirsel[g][3], sel1 = dirsel[g + 8][3];
    if (q == 0 && A.out.sigma) {
        if (row0 + g < n) A.out.sigma[row0 + g] = expf(b1acc[0][0]) * sel0;
        if (row0 + g + 8 < n) A.out.sigma[row0 + g + 8] = expf(b1acc[0][2]) * sel1;
    }
    if (!HEAD) return;
    uint32_t ha[2][4];
    {
        float g00 = b1acc[0][0], g02 = b1acc[0][2];
        if (q == 0) { g00 = 1.0f; g02 = 1.0f; }
        ha[0][0] = pack_h2(g00, b1acc[0][1]);
        ha[0][1] = pack_h2(g02, b1acc[0][3]);
        ha[0][2] = pack_h2(b1acc[1][0], b1acc[1][1]);
        ha[0][3] = pack_h2(b1acc[1][2], b1acc[1][3]);
        float e[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = g + 8 * h;
            const float d0 = (dirsel[r][0] + 1.0f) / 2.0f, d1 = (dirsel[r][1] + 1.0f) / 2.0f,
                        d2 = (dirsel[r][2] + 1.0f) / 2.0f;
            e[h][0] = q == 0 ? d0 : (q == 1 ? d2 : 1.0f);
            e[h][1] = q == 0 ? d1 : 1.0f;
        }
        ha[1][0] = pack_h2(e[0][0], e[0][1]);
        ha[1][1] = pack_h2(e[1][0], e[1][1]);
        ha[1][2] = pack_h2(1.0f, 1.0f);
        ha[1][3] = pack_h2(1.0f, 1.0f);
    }
    float c0acc[8][4];
    smem_gemm<2, 4>(c0acc, ha, field_w + 384, lane);
    uint32_t c1in[4][4];
    relu_pack_nobias<8>(c0acc, c1in);
    float c1acc[8][4];
    smem_gemm<4, 4>(c1acc, c1in, field_w + 640, lane);
    uint32_t c2in[4][4];
    relu_pack_nobias<8>(c1acc, c2in);
    float c2acc[2][4];
    smem_gemm<4, 1>(c2acc, c2in, field_w + 1152, lane);
    if (A.out.rgb) {
        const int64_t sa = row0 + g, sb = row0 + g + 8;
        if (q == 0) {
            if (sa < n) { A.out.rgb[3 * sa + 0] = 1.f / (1.f + expf(-c2acc[0][0])); A.out.rgb[3 * sa + 1] = 1.f / (1.f + expf(-c2acc[0][1])); }
            if (sb < n) { A.out.rgb[3 * sb + 0] = 1.f / (1.f + expf(-c2acc[0][2])); A.out.rgb[3 * sb + 1] = 1.f / (1.f + expf(-c2acc[0][3])); }
        } else if (q == 1) {
            if (sa < n) A.out.rgb[3 * sa + 2] = 1.f / (1.f + expf(-c2acc[0][0]));
            if (sb < n) A.out.rgb[3 * sb + 2] = 1.f / (1.f + expf(-c2acc[0][2]));
        }
    }
}

// SAVE: training instantiation, additionally stores the warped positions and the deformation activations the
// backward kernels read; compiled out of the inference instantiation (the stores cost ~40 B of spills there).
template <bool DEFORM, bool FIELD, bool HEAD, bool SAVE>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) field_kernel_ws(const __grid_constant__ FieldArgs A) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemWS &sm = *reinterpret_cast<SmemWS *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr bool FEAT_GIVEN = false, LERP = false;
    // NOTE: nothing is computed ahead of the role split on purpose.  Values shared by both roles get registers that
    // suit the 88-register tensor role, and the 64-register gather role then pays for them with spills inside its
    // sample loop.  Each role derives its loop bounds itself.

#define NSB_N_SAMPLES A.S.n_samples
#include "nsb_field_setup.inc"
    if (warp >= kTensorWarps) {
        // =============================== GATHER warps ===============================
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
#include "nsb_field_gather_role.inc"
        return;
    }

    // =============================== TENSOR warps ===============================
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
#include "nsb_field_tensor_role.inc"
#undef NSB_N_SAMPLES
}

// Training forward over the KEPT samples when the density pre-pass already gathered their features (SURVEY 8(f)-1:
// "reuse the pre-pass evaluation"): deformation MLP (activations saved for the backward) + density / colour MLPs from
// nsb_samples.given_feat; the gather warps exit at once -- no table line is read a second time.
template <bool DEFORM>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) field_kernel_ws_given(const __grid_constant__ FieldArgs A) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemWS &sm = *reinterpret_cast<SmemWS *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr bool FIELD = true, HEAD = true, SAVE = true, FEAT_GIVEN = true, LERP = false;
#define NSB_N_SAMPLES A.S.n_samples
#include "nsb_field_setup.inc"
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
#include "nsb_field_gather_role.inc"
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
#include "nsb_field_tensor_role.inc"
#undef NSB_N_SAMPLES
}

// ===========================================================================================
// wgmma variant of the inference kernels ("tc" kernels): the deformation MLP as warpgroup MMAs (accumulator in
// registers, weights read from shared memory by the tensor core once per 64-row half of a 128-row tile) --
// nsb_field_tensor_role_tc.inc.  The gather role is the unchanged include; only the tensor role and the shared-memory
// plan differ.
// ===========================================================================================
constexpr int kFrameGatherWarps = 8;   // frame-table gather: how many of the gather warps do work
constexpr int kTcStages = 4, kTcBlocksPerTile = 14;
#ifdef NSB_TC_PROF
constexpr int kTcProfPhases = 10;    // tools/tc_prof.py names them
__device__ unsigned long long g_tc_prof[kTcProfPhases], g_tc_prof_k[8];
#define KPROF(i) if (threadIdx.x == 0 && blockIdx.x == 3) g_tc_prof_k[i] = (unsigned long long)clock64();
#else
#define KPROF(i)
#endif
constexpr size_t kTcPackedBytes = 12 * 16384 + 2 * 2048;

// Warp index that ptxas can see is uniform across the warp (lane 0's value, broadcast).  With `tid >> 5`, ptxas cannot
// prove that the role split `warp < kTensorWarps` keeps whole warpgroups together, inserts a warpgroup arrive in the
// divergent path and serialises every wgmma.mma_async of the deformation chain (ptxas C7520).  The *_ws kernels keep
// `tid >> 5`: there the broadcast moves their gather-role register allocation and adds spills in the sample loop.
__device__ __forceinline__ int tc_warp_index(int tid) { return __shfl_sync(0xffffffffu, tid >> 5, 0); }

// Code-bias rows deform_code_bias[t][0|1][128] (fp32, 1 KB per timestep) staged in shared memory for the epilogues of
// layers 0 and 4 of the frame-table kernels.  Up to kTcCodeBiasRows timesteps are staged; a larger table is read from
// global memory (tc_code_bias_rows).  The rows sit over blend_b / cv_stage, which the frame gather role never touches;
// the launch sizes the dynamic shared memory from T.
constexpr int kTcCodeBiasRows = 32;
constexpr int kTcBiasFloats = 4 * 128 + 8;      // sm.bias: the biases of layers 1, 2, 3, 5, then the heads (v 0..2, r 3..5)

struct alignas(1024) SmemTC {
    uint8_t wring[kTcStages][16384];        // weight blocks [128 n x 64 k] (heads: [16 x 64]) in core-matrix order
    uint8_t a_enc[12288];                   // posenc A operand [128 rows x 48 k] (the hidden layers' A stays in registers)
    uint4 field_w[kFieldPackedU4];
    alignas(16) float bias[kTcBiasFloats];  // layers 0 and 4 take their bias from the code-bias rows
    alignas(16) float heads[2][64][8];      // deformation head outputs (v 0..2, r 3..5) of each warpgroup's 64 rows
    uint64_t full[kTcStages];
    uint64_t xs_full[2], feat_full[2];
    uint32_t ring_rel[kTcStages];           // releases of each weight-ring stage by the 8 tensor warps (8 per use)
    int row_ts[NSB_TILE];                   // timestep of each row of the tile in flight (its code-bias row)
    int tile_ctr[2];
    int64_t n_dyn;
    uint64_t sampler_done;
    alignas(16) float xs[2][NSB_TILE][4];
    alignas(16) __half feat[2][NSB_TILE * kFeatStride];
    alignas(16) float dirsel[2][NSB_TILE][4];
    uint2 blend_b[kGatherWarps][4 * 32];    // per-sample blend only
    uint4 cv_stage[kGatherWarps][1];        // SAVE is never instantiated with the tc role; the gather include names it
};
// byte offset of the staged code-bias rows in dynamic shared memory (a multiple of 128: the swizzle of NSB_TC_SETUP
// permutes 32-byte chunks inside 128-byte lines), and the dynamic shared memory of a launch
template <bool FRAME>
__host__ __device__ constexpr size_t tc_code_bias_offset() {
    return (FRAME ? offsetof(SmemTC, blend_b) + 127 : offsetof(SmemTC, cv_stage) + sizeof(SmemTC::cv_stage) + 127) / 128 * 128;
}
template <bool FRAME>
__host__ __device__ constexpr size_t tc_smem_bytes(int staged_rows) { return tc_code_bias_offset<FRAME>() + (size_t)staged_rows * 1024; }
static_assert(tc_code_bias_offset<true>() % 128 == 0 && tc_code_bias_offset<false>() % 128 == 0, "code-bias swizzle");
static_assert(tc_smem_bytes<false>(kTcCodeBiasRows) <= 227 * 1024, "shared memory plan");
// Frame-table kernels: with every T <= kTcCodeBiasRows staged, the kernel (+ 1 KB reserved per CTA) still fits H100's
// 164 KB shared-memory carveout step, which leaves the gather role ~92 KB of L1.
static_assert(tc_smem_bytes<true>(kTcCodeBiasRows) + 1024 <= 164 * 1024, "frame-table kernels: 164 KB carveout step");
static_assert(kTensorWarps == 8, "the wgmma tensor role runs two warpgroups of 64 rows");
// timesteps whose code-bias rows a tc launch stages in shared memory: all of them, or none (global fallback).  The
// per-sample blend kernels (!FRAME) are bound by their gather role and read the global table.
template <bool FRAME>
__host__ __device__ __forceinline__ int tc_code_bias_rows(int n_timesteps) {
    return FRAME && n_timesteps <= kTcCodeBiasRows ? n_timesteps : 0;
}

// setup shared by the tc kernels (textual for the same reason as the other role bodies).  The code-bias rows are stored
// swizzled: the 32-byte chunk c (columns 8c .. 8c + 7) of timestep t's row moves to chunk c ^ (t & 3), so the 8 rows of
// an epilogue load (8 timesteps at a 1 KB stride, which would all hit the same 8 banks) spread over the 4 bank groups.
#define NSB_TC_SETUP()                                                                                              \
    {                                                                                                               \
        const uint4 *src = reinterpret_cast<const uint4 *>(A.P.field_packed);                                      \
        for (int i = tid; i < kFieldPackedU4; i += kThreadsWS) sm.field_w[i] = __ldg(src + i);                     \
        for (int i = tid; i < kTcBiasFloats; i += kThreadsWS)                                                      \
            sm.bias[i] = __ldg(A.P.deform_bias + (i < 3 * 128 ? 128 + i : 256 + i));   /* skip layers 0, 4 */    \
        for (int i = tid; i < (int)(sizeof(sm.a_enc) / 16); i += kThreadsWS) reinterpret_cast<uint4 *>(&sm.a_enc)[i] = make_uint4(0u, 0u, 0u, 0u); \
        {                                                                                                           \
            float *const cb_s = reinterpret_cast<float *>(smem_raw + tc_code_bias_offset<FRAME>());                \
            const float4 *cb_g = reinterpret_cast<const float4 *>(A.P.deform_code_bias);                           \
            for (int i = tid; i < tc_code_bias_rows<FRAME>(A.P.n_timesteps) * 64; i += kThreadsWS) {                      \
                const int t = i >> 6, c = (i >> 1) & 15;     /* 4 floats: row t, layer (i >> 5) & 1, chunk c */    \
                *reinterpret_cast<float4 *>(cb_s + t * 256 + ((i >> 5) & 1) * 128 + (c ^ (t & 3)) * 8 + (i & 1) * 4) = __ldg(cb_g + i); \
            }                                                                                                       \
        }                                                                                                           \
        if (tid == 0) {                                                                                             \
            for (int s = 0; s < kTcStages; ++s) { mbar_init(&sm.full[s], 1); sm.ring_rel[s] = 0; }                \
            for (int b = 0; b < 2; ++b) {                                                                           \
                mbar_init(&sm.xs_full[b], kTensorWarps);                                                            \
                mbar_init(&sm.feat_full[b], kGatherWarps);                                                          \
                sm.tile_ctr[b] = 0;                                                                                 \
            }                                                                                                       \
            mbar_fence_init();                                                                                      \
        }                                                                                                           \
        __syncthreads();                                                                                            \
    }

// FRAME: the gather role reads the member-blended frame table (nsb_field_gather_role_frame.inc); STACK: one table per
// timestep (frame_stride != 0).  STACK is a template flag so that the single-frame kernels compile exactly as without the
// timestep offset: ptxas' allocation of the whole kernel (tensor role included) moves with any change to the gather code.
template <bool HEAD, bool FRAME, bool STACK>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) field_kernel_tc(const __grid_constant__ FieldArgs A) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemTC &sm = *reinterpret_cast<SmemTC *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tc_warp_index(tid);
    constexpr bool FIELD = true, SAVE = false, FEAT_GIVEN = false, LERP = false;
#define NSB_N_SAMPLES A.S.n_samples
    NSB_TC_SETUP()
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
        if constexpr (FRAME) {
#include "nsb_field_gather_role_frame.inc"
        } else {
#include "nsb_field_gather_role.inc"
        }
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
#include "nsb_field_tensor_role_tc.inc"
#undef NSB_N_SAMPLES
}

// field_kernel_ws with the sample count read from DEVICE memory (nsb_samples.n_samples_dev; the sync-free training
// sampler: the host never learns how many candidates the march produced).  grid = number of SMs; A.S.n_samples is the
// capacity of the sample arrays.  Same role bodies.
template <bool DEFORM, bool FIELD, bool HEAD, bool SAVE>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) field_kernel_ws_dyn(const __grid_constant__ FieldArgs A) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemWS &sm = *reinterpret_cast<SmemWS *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr bool FEAT_GIVEN = false, LERP = false;
    if (tid == 0) sm.n_dyn = min(*A.S.n_samples_dev, A.S.n_samples);      // visible after the setup's __syncthreads
#define NSB_N_SAMPLES (*reinterpret_cast<const volatile int64_t *>(&sm.n_dyn))
#include "nsb_field_setup.inc"
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
#include "nsb_field_gather_role.inc"
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
#include "nsb_field_tensor_role.inc"
#undef NSB_N_SAMPLES
}

// ===========================================================================================
// render_kernel_ws: sampler -> field -> composite in ONE launch (north star: "fused into one kernel").
// A persistent cooperative kernel, one CTA per SM, whose phases are separated by grid-wide barriers:
//   S  sampler.  Fixed stride: one warp per ray (march_fixed_warp).  Occupancy grid (nerfacc traverse_grids): the
//      samples come from march_occ_coop_kernel (nsb_render.cu), launched just before, and the phase reads their count
//      from the workspace header.  The packed sample count stays on the device (shared-memory word n_dyn): no host
//      synchronisation.
//   F  the field phase = the body of field_kernel_ws, textually (same setup / gather role / tensor role includes).
//   C  compositing by the tensor warps (composite_ray, one warp per ray) | barrier | global depth clip.
// Per-sample sigma / rgb / offsets cross from F to C through the caller's workspace (32 B per sample: L2-resident
// at 2^20 samples, 0.2 % of the gather traffic).  Every phase runs the device code of the stand-alone kernels, so the
// results are bit-identical to nsb_march_* + nsb_field_forward + nsb_composite_forward.
// ===========================================================================================
struct RenderKArgs {
    FieldArgs F;              // S.* and out.* point into the caller's workspace
    nsb_march_args M;         // occupancy sampler (counts / offsets / outputs in the workspace)
    nsb_composite_args C;
    int32_t sampler, n_per_ray;
    float near_plane;
    int64_t capacity;
    nsb_render_ws_header *hdr;
    int64_t *partials;        // [gridDim.x] chunk sums of the ray-count scan
    int64_t *packed_info;     // [n_rays][2] out (C.packed_info is the same buffer, const)
};

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// Grid-wide barrier of the tensor warps (the only warps that run the sampler / compositing phases): one leader thread
// per CTA on a global arrival counter (cooperative launch: all CTAs are resident).  `target` = arrivals expected so
// far = (barrier index + 1) * gridDim.x; the counter is zeroed by the host before the launch.
__device__ __forceinline__ void phase_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kTensorWarps * 32) : "memory"); }
__device__ __forceinline__ void grid_barrier(uint32_t *ctr, const uint32_t target) {
    phase_sync();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        while (ld_acquire_u32(ctr) < target) __nanosleep(40);
        __threadfence();
    }
    phase_sync();
}

// Where the extra phases run.  The 64-register gather role is allocated erratically by ptxas: with the sampler phase
// inline, or as a call ahead of the role split, it went from 1 to 37-82 spill instructions (tools/spill_report.py;
// a spill in the sample loop costs more than everything this kernel saves).  So BOTH extra phases run on the TENSOR
// warps, as calls after the role split: the gather warps' code is the text of field_kernel_ws plus one named barrier
// on which they wait for the sampler (and the sample count in shared memory) before their first tile.
constexpr int kPhaseThreads = kTensorWarps * 32;

// SAMPLER: 0 fixed-stride march fused; 2 samples GIVEN: a preceding launch (march_occ_coop_kernel, nsb_render.cu) filled
// the packed arrays and left the count in the workspace header; 4 either of the two, chosen at run time by K.sampler.
// the fixed-stride march of this CTA's rays as a real call (tensor warps, after the role split)
__device__ __noinline__ void fixed_march_rays(const RenderKArgs &K, const int warp, const int lane) {
    const int64_t R = K.C.n_rays;
    for (int64_t r = (int64_t)blockIdx.x * kTensorWarps + warp; r < R; r += (int64_t)gridDim.x * kTensorWarps) {
        const float t0 = march_fixed_t0(K.F.S.origins, K.F.S.directions, K.F.P.aabb, r, K.near_plane);
        march_fixed_warp(t0, r, K.n_per_ray, K.M.step, K.M.t_starts, K.M.t_ends, K.M.ray_indices, lane);
        if (lane == 0) { K.packed_info[2 * r] = r * K.n_per_ray; K.packed_info[2 * r + 1] = K.n_per_ray; }
    }
}

template <int SAMPLER, class SM = SmemWS>
__device__ __forceinline__ void render_sampler_phase(const RenderKArgs &K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SM &sm = *reinterpret_cast<SM *>(smem_raw);
    const FieldArgs &A = K.F;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;      // tid < kPhaseThreads
    uint32_t *const bar = &K.hdr->barrier;
    const int64_t R = K.C.n_rays;
    if (blockIdx.x == 0 && tid == 0) {
        K.hdr->depth_range[0] = 0xffffffffu;
        K.hdr->depth_range[1] = 0u;
        if (SAMPLER != 2 && !(SAMPLER == 4 && K.sampler != 0)) K.hdr->status = 0;
    }
    if constexpr (SAMPLER == 4) {
        // run-time choice between the fixed march and given samples in ONE binary (the wgmma render kernel): two
        // instantiations are two draws of ptxas' allocation of the gather role
        if (K.sampler == 0) {
            fixed_march_rays(K, warp, lane);
            if (tid == 0) {
                sm.n_dyn = R * K.n_per_ray;
                if (blockIdx.x == 0) K.hdr->n_total = R * K.n_per_ray;
            }
        } else if (tid == 0) {
            sm.n_dyn = min(__ldcg(&K.hdr->n_total), K.capacity);
        }
        grid_barrier(bar, 1u * gridDim.x);
    } else if constexpr (SAMPLER == 2) {
        if (tid == 0) sm.n_dyn = min(__ldcg(&K.hdr->n_total), K.capacity);
        grid_barrier(bar, 1u * gridDim.x);          // depth_range initialised before any CTA composites
    } else {
        for (int64_t r = (int64_t)blockIdx.x * kTensorWarps + warp; r < R; r += (int64_t)gridDim.x * kTensorWarps) {
            const float t0 = march_fixed_t0(A.S.origins, A.S.directions, A.P.aabb, r, K.near_plane);
            march_fixed_warp(t0, r, K.n_per_ray, K.M.step, K.M.t_starts, K.M.t_ends, K.M.ray_indices, lane);
            if (lane == 0) { K.packed_info[2 * r] = r * K.n_per_ray; K.packed_info[2 * r + 1] = K.n_per_ray; }
        }
        if (tid == 0) {
            sm.n_dyn = R * K.n_per_ray;     // the host sized the workspace for exactly this
            if (blockIdx.x == 0) K.hdr->n_total = R * K.n_per_ray;
        }
        grid_barrier(bar, 1u * gridDim.x);
    }
}

// the grid barriers continue the count of render_sampler_phase, which ended with barrier 1
__device__ __forceinline__ void render_composite_phase(const RenderKArgs &K) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t *const bar = &K.hdr->barrier;
    const int64_t R = K.C.n_rays;
    grid_barrier(bar, 2u * gridDim.x);
    for (int64_t ray = (int64_t)blockIdx.x * kTensorWarps + warp; ray < R; ray += (int64_t)gridDim.x * kTensorWarps)
        composite_ray(K.C, ray, lane);
    grid_barrier(bar, 3u * gridDim.x);
    {   // DepthRenderer('expected'): clip to the global [min, max] of the sample midpoints
        const uint32_t lo_u = __ldcg(&K.hdr->depth_range[0]), hi_u = __ldcg(&K.hdr->depth_range[1]);
        // no sample in the whole batch: the reference inserts one fake sample with t_start = t_end = 1 on ray 0
        // (nersemble_volumetric_sampler.py:110-114), whose midpoint clips every ray's depth (0) to 1
        const float lo = lo_u != 0xffffffffu ? ordered_to_float(lo_u) : 1.0f, hi = lo_u != 0xffffffffu ? ordered_to_float(hi_u) : 1.0f;
        for (int64_t r = (int64_t)blockIdx.x * kPhaseThreads + tid; r < R; r += (int64_t)gridDim.x * kPhaseThreads)
            K.C.out_depth[r] = fminf(fmaxf(K.C.out_depth[r], lo), hi);
    }
}

template <bool DEFORM, int SAMPLER>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) render_kernel_ws(const __grid_constant__ RenderKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemWS &sm = *reinterpret_cast<SmemWS *>(smem_raw);
    const FieldArgs &A = K.F;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr bool FIELD = true, HEAD = true, SAVE = false, FEAT_GIVEN = false, LERP = false;

#define NSB_N_SAMPLES (*reinterpret_cast<const volatile int64_t *>(&sm.n_dyn))
    if (tid == 0) mbar_init(&sm.sampler_done, 1);                          // fenced + published by the setup below
#include "nsb_field_setup.inc"
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
        mbar_wait<200>(&sm.sampler_done, 0);                               // the sampler is done, sm.n_dyn is set
#include "nsb_field_gather_role.inc"
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
    render_sampler_phase<SAMPLER>(K);                                      // S (ends with a grid barrier)
    // hand-off through an mbarrier rather than a named barrier shared by the two roles: compute-sanitizer synccheck
    // reports a barrier that warps reach from two different instructions as divergent
    if (tid == 0) mbar_arrive(&sm.sampler_done);
    {
#include "nsb_field_tensor_role.inc"
    }
#undef NSB_N_SAMPLES
    render_composite_phase(K);                                             // C
}

// render_kernel_ws with the deformation MLP on wgmma (nsb_field_tensor_role_tc.inc); SAMPLER 2 or 4
template <int SAMPLER, bool FRAME, bool STACK>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) render_kernel_tc(const __grid_constant__ RenderKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemTC &sm = *reinterpret_cast<SmemTC *>(smem_raw);
    const FieldArgs &A = K.F;
    const int tid = threadIdx.x, lane = tid & 31, warp = tc_warp_index(tid);
    constexpr bool FIELD = true, HEAD = true, SAVE = false, FEAT_GIVEN = false, LERP = false;
#define NSB_N_SAMPLES (*reinterpret_cast<const volatile int64_t *>(&sm.n_dyn))
    KPROF(0)
    if (tid == 0) mbar_init(&sm.sampler_done, 1);
    NSB_TC_SETUP()
    KPROF(1)
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
        mbar_wait<200>(&sm.sampler_done, 0);
        if constexpr (FRAME) {
#include "nsb_field_gather_role_frame.inc"
        } else {
#include "nsb_field_gather_role.inc"
        }
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
    render_sampler_phase<SAMPLER, SmemTC>(K);
    KPROF(2)
    if (tid == 0) mbar_arrive(&sm.sampler_done);
    {
#include "nsb_field_tensor_role_tc.inc"
    }
#undef NSB_N_SAMPLES
    KPROF(3)
    render_composite_phase(K);
    KPROF(4)
}

// render_kernel_tc at continuous ray times (nsb_render_forward_interp, DESIGN 4.2g): the same role bodies with LERP set.
// Every row carries its fractional timestep u (sample_time_u) in xs.w and row_ts instead of its timestep; the gather
// interpolates the stack entries (FRAME = STACK = true) or the blend codes (FRAME = STACK = false) of floor(u) and
// floor(u) + 1, the tensor role the code-bias rows of layers 0 and 4.  Its own name: a fourth template flag on
// render_kernel_tc would give the existing kernels new symbols.
template <int SAMPLER, bool FRAME, bool STACK>
__global__ void __launch_bounds__(kLaunchBoundWS, 1) render_kernel_tc_lerp(const __grid_constant__ RenderKArgs K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SmemTC &sm = *reinterpret_cast<SmemTC *>(smem_raw);
    const FieldArgs &A = K.F;
    const int tid = threadIdx.x, lane = tid & 31, warp = tc_warp_index(tid);
    constexpr bool FIELD = true, HEAD = true, SAVE = false, FEAT_GIVEN = false, LERP = true;
    static_assert(FRAME == STACK, "linear time: the timestep stack or the per-sample blend");
#define NSB_N_SAMPLES (*reinterpret_cast<const volatile int64_t *>(&sm.n_dyn))
    if (tid == 0) mbar_init(&sm.sampler_done, 1);
    NSB_TC_SETUP()
    if (warp >= kTensorWarps) {
        if (kGatherRegs != kLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGatherRegs));
        mbar_wait<200>(&sm.sampler_done, 0);
        if constexpr (FRAME) {
#include "nsb_field_gather_role_frame.inc"
        } else {
#include "nsb_field_gather_role.inc"
        }
        return;
    }
    if (kTensorRegs != kLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTensorRegs));
    render_sampler_phase<SAMPLER, SmemTC>(K);
    if (tid == 0) mbar_arrive(&sm.sampler_done);
    {
#include "nsb_field_tensor_role_tc.inc"
    }
#undef NSB_N_SAMPLES
    render_composite_phase(K);
}

// -------------------------------------------------------------------------------------------
// stand-alone HashEnsemble.forward (component API): one warp per sample, grid-stride
// -------------------------------------------------------------------------------------------
struct HashArgs {
    nsb_field_params P;
    nsb_field_opts O;
    const float *x;
    const float *codes;
    int64_t n;
    void *out;
    int out_is_half;
};

__global__ void __launch_bounds__(256) hash_blend_kernel(const __grid_constant__ HashArgs H) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t s = warp_global; s < H.n; s += n_warps) {
        const float x = H.x[3 * s + 0], y = H.x[3 * s + 1], z = H.x[3 * s + 2];
        const int mg = lane & 7;
        float4 c = __ldg(reinterpret_cast<const float4 *>(H.codes + s * NSB_MEMBERS) + mg);
        float cw[4];
        cw[0] = fmaf(c.x, H.O.cw_scale[4 * mg + 0], H.O.cw_bias[4 * mg + 0]);
        cw[1] = fmaf(c.y, H.O.cw_scale[4 * mg + 1], H.O.cw_bias[4 * mg + 1]);
        cw[2] = fmaf(c.z, H.O.cw_scale[4 * mg + 2], H.O.cw_bias[4 * mg + 2]);
        cw[3] = fmaf(c.w, H.O.cw_scale[4 * mg + 3], H.O.cw_bias[4 * mg + 3]);
        const float val = gather_blend<2>(H.P, x, y, z, cw, lane);
        if (H.out_is_half)
            reinterpret_cast<__half *>(H.out)[s * 32 + lane] = __float2half_rn(val);
        else
            reinterpret_cast<float *>(H.out)[s * 32 + lane] = val;
    }
}

// -------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------
constexpr size_t kRenderHdrBytes = 64, kRenderPartials = 1024;
static_assert(sizeof(nsb_render_ws_header) == kRenderHdrBytes, "workspace header layout");

// Launch of a persistent kernel (kThreadsWS threads per CTA).  The kernel's dynamic shared-memory limit is raised to
// max_smem on its first launch.  coop_barrier != nullptr makes it a cooperative launch (the render kernels: their grid
// barriers need every CTA resident) whose barrier counter *coop_barrier is zeroed first.
template <auto Kernel, class Args>
static int launch_persistent(const Args &a, size_t smem, size_t max_smem, int grid, uint32_t *coop_barrier,
                             const char *name, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%s): %s", name, cudaGetErrorString(e)); return 1; }
        configured = true;
    }
    if (!coop_barrier) {
        Kernel<<<grid, kThreadsWS, smem, st>>>(a);
        return check_launch(name);
    }
    if ((size_t)grid > kRenderPartials) { set_error("nsb_render_forward: more SMs than scan partials"); return 1; }
    cudaError_t e = cudaMemsetAsync(coop_barrier, 0, sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("nsb_render_forward: memset: %s", cudaGetErrorString(e)); return 2; }
    void *kargs[] = {const_cast<Args *>(&a)};
    e = cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(Kernel), dim3(grid), dim3(kThreadsWS), kargs, smem, st);
    if (e != cudaSuccess) { set_error("%s: %s", name, cudaGetErrorString(e)); return 2; }
    return check_launch(name);
}

// grid of the field kernels: one CTA per tile, at most one per SM
static int field_grid(const FieldArgs &A) {
    const int64_t n_tiles = (A.S.n_samples + NSB_TILE - 1) / NSB_TILE;
    return (int)std::min<int64_t>(n_tiles, (int64_t)num_sms());
}

template <bool D, bool F, bool H>
static int launch_field_ws(const FieldArgs &A, cudaStream_t st) {
    const bool save = A.out.xs || A.out.deform_acts || A.out.deform_enc || A.out.corner_vals;
    constexpr size_t smem = sizeof(SmemWS);
    return save ? launch_persistent<field_kernel_ws<D, F, H, true>>(A, smem, smem, field_grid(A), nullptr, "field_kernel_ws", st)
                : launch_persistent<field_kernel_ws<D, F, H, false>>(A, smem, smem, field_grid(A), nullptr, "field_kernel_ws", st);
}

// The tc role takes every row's code bias from the per-timestep table (staged in shared memory up to
// kTcCodeBiasRows timesteps): calls with per-sample code bias (the component API's sample_warp_codes) run the *_ws
// kernels (launch_field), and the fused render never sets one.
static bool tc_args_ok(const FieldArgs &A) {
    if (A.S.sample_code_bias || !A.P.deform_code_bias) {
        set_error("tc kernels: the code bias must come from the per-timestep table deform_code_bias");
        return false;
    }
    return true;
}

template <bool H, bool FR, bool ST>
static int launch_field_tc_(const FieldArgs &A, cudaStream_t st) {
    if (!tc_args_ok(A)) return 1;
    return launch_persistent<field_kernel_tc<H, FR, ST>>(A, tc_smem_bytes<FR>(tc_code_bias_rows<FR>(A.P.n_timesteps)),
                                                         tc_smem_bytes<FR>(tc_code_bias_rows<FR>(kTcCodeBiasRows)),
                                                         field_grid(A), nullptr, "field_kernel_tc", st);
}
template <bool H>
static int launch_field_tc(const FieldArgs &A, cudaStream_t st) {
    if (!A.P.frame_table) return launch_field_tc_<H, false, false>(A, st);
    return A.P.frame_stride ? launch_field_tc_<H, true, true>(A, st) : launch_field_tc_<H, true, false>(A, st);
}

template <bool D, bool F, bool H>
static int launch_field(const FieldArgs &A, cudaStream_t st) {
    constexpr size_t smem = sizeof(SmemWS);
    if (A.S.given_feat) {
        if (F && H && !A.S.n_samples_dev)
            return launch_persistent<field_kernel_ws_given<D>>(A, smem, smem, field_grid(A), nullptr, "field_kernel_ws_given", st);
        set_error("nsb_field_forward: given_feat needs the full evaluation (rgb) and a host-side sample count");
        return 1;
    }
    if (A.S.n_samples_dev) {
        // device-side sample count: the density pre-pass of the training sampler (each instantiation costs ~15 s of
        // ptxas).  Always the SAVE instantiation (its stores are skipped at run time when the pointers are NULL): ptxas
        // gives its gather role 0 spill instructions, the non-SAVE density instantiation 37 (tools/spill_report.py)
        if (F && !H)
            return launch_persistent<field_kernel_ws_dyn<D, true, false, true>>(A, smem, smem, field_grid(A), nullptr,
                                                                                "field_kernel_ws_dyn", st);
        set_error("nsb_field_forward: n_samples_dev is supported for the density evaluation (no rgb) only");
        return 1;
    }
    if (D && F && A.P.deform_packed_umma && !A.S.sample_code_bias && !(A.out.xs || A.out.deform_acts || A.out.deform_enc || A.out.corner_vals || A.out.feat))
        return launch_field_tc<H>(A, st);       // inference with the deformation MLP on wgmma
    return launch_field_ws<D, F, H>(A, st);
}

}  // namespace nsb

using namespace nsb;

extern "C" size_t nsb_deform_packed_bytes(void) { return (size_t)kTbNumSlabs * kSlabBytes; }
extern "C" size_t nsb_field_packed_bytes(void) { return kFieldPackedU4 * sizeof(uint4); }
extern "C" size_t nsb_deform_packed_umma_bytes(void) { return kTcPackedBytes; }
#ifdef NSB_TC_PROF
extern "C" int nsb_debug_tc_prof(unsigned long long *out) {      // kTcProfPhases cycle counters
    return (int)cudaMemcpyFromSymbol(out, nsb::g_tc_prof, sizeof(unsigned long long) * kTcProfPhases);
}
extern "C" int nsb_debug_tc_prof_kernel(unsigned long long *out8) {      // clock64 at the phase boundaries of render_kernel_tc
    return (int)cudaMemcpyFromSymbol(out8, nsb::g_tc_prof_k, sizeof(unsigned long long) * 8);
}
#endif

extern "C" int nsb_field_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                 const nsb_field_out *out, void *stream) {
    if (!params || !opts || !samples || !out) { set_error("nsb_field_forward: null argument"); return 1; }
    if (samples->n_samples <= 0) return 0;
    if (check_field_params("nsb_field_forward", params) || check_samples("nsb_field_forward", samples)) return 1;
    const bool deform = opts->use_deformation != 0;
    const bool need_field = out->sigma || out->rgb || out->feat || out->xs;
    const bool head = opts->compute_rgb != 0 && out->rgb != nullptr;
    if (!need_field && !(deform && out->offsets)) { set_error("nsb_field_forward: no outputs requested"); return 1; }
    if (need_field && (!params->tables || !params->field_packed)) { set_error("nsb_field_forward: tables/field_packed missing"); return 1; }
    if (need_field && !params->blend_codes && !samples->sample_blend_codes) { set_error("nsb_field_forward: no blend codes"); return 1; }
    if (deform && (!params->deform_packed_tb || !params->deform_bias || (!params->deform_code_bias && !samples->sample_code_bias))) {
        set_error("nsb_field_forward: deformation parameters missing (deform_packed_tb, deform_bias, code bias)");
        return 1;
    }
    if (deform && samples->sample_code_bias && (samples->n_samples > (int64_t(1) << 24) || (need_field && !samples->sample_blend_codes))) {
        set_error("nsb_field_forward: per-sample code bias needs <= 2^24 samples and per-sample blend codes");
        return 1;
    }
    FieldArgs A;
    A.P = *params; A.O = *opts; A.S = *samples; A.out = *out;
    for (int k = 0; k < 3; ++k) A.aabb_size[k] = params->aabb[3 + k] - params->aabb[k];
    cudaStream_t st = (cudaStream_t)stream;
    if (deform) {
        if (!need_field) return launch_field<true, false, false>(A, st);
        return head ? launch_field<true, true, true>(A, st) : launch_field<true, true, false>(A, st);
    }
    return head ? launch_field<false, true, true>(A, st) : launch_field<false, true, false>(A, st);
}

extern "C" int nsb_hash_blend_forward(const nsb_field_params *params, const nsb_field_opts *opts, const float *x,
                                      const float *codes, int64_t n, void *out, int32_t out_is_half, void *stream) {
    if (!params || !opts || !x || !codes || !out) { set_error("nsb_hash_blend_forward: null argument"); return 1; }
    if (n <= 0) return 0;
    if (params->levels.n_levels != NSB_MAX_LEVELS) { set_error("nsb_hash_blend_forward: n_levels must be 16"); return 1; }
    HashArgs H;
    H.P = *params; H.O = *opts; H.x = x; H.codes = codes; H.n = n; H.out = out; H.out_is_half = out_is_half;
    const int64_t warps_needed = n;
    const int blocks = (int)std::min<int64_t>((warps_needed + 7) / 8, (int64_t)num_sms() * 8);
    hash_blend_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(H);
    return check_launch("hash_blend_kernel");
}

// -------------------------------------------------------------------------------------------
// nsb_blend_tables: frame tables = the 32 members of every table entry blended with the weights of n_ts consecutive
// timesteps (cw[t][m] = code[t][m] * cw_scale[m] + cw_bias[m], hash_ensemble.py:119-139), float2 per entry and timestep.
// 8 lanes per entry (16 B = 4 members each), fp32 accumulation, the same member order and xor tree for every timestep;
// one streaming pass over the tables (each 128 B line read once for all timesteps; the weights sit in shared memory).
// -------------------------------------------------------------------------------------------
namespace nsb {
constexpr int kBlendMaxTimesteps = 256;        // 32 KB of weights in shared memory
__global__ void __launch_bounds__(256) blend_tables_kernel(const uint4 *__restrict__ tables, const float *__restrict__ code,
                                                           const __grid_constant__ nsb_field_opts O, float2 *__restrict__ out,
                                                           int n_ts, int64_t n_entries) {
    __shared__ float4 cw_s[kBlendMaxTimesteps][8];
    const int lane = threadIdx.x & 31, sub = lane & 7;
    for (int i = threadIdx.x; i < n_ts * 8; i += blockDim.x) {
        const int t = i >> 3, s = i & 7;
        float cw[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) cw[k] = fmaf(__ldg(code + t * NSB_MEMBERS + 4 * s + k), O.cw_scale[4 * s + k], O.cw_bias[4 * s + k]);
        cw_s[t][s] = make_float4(cw[0], cw[1], cw[2], cw[3]);
    }
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * (blockDim.x >> 3);
    for (int64_t e = (int64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3); e < ((n_entries + 3) & ~(int64_t)3); e += stride) {
        float2 f[4] = {};
        if (e < n_entries) {
            const uint4 v = __ldcs(tables + e * 8 + sub);          // streamed once: evict-first
            f[0] = unpack_h2(v.x); f[1] = unpack_h2(v.y); f[2] = unpack_h2(v.z); f[3] = unpack_h2(v.w);
        }
        for (int t = 0; t < n_ts; ++t) {
            const float4 c4 = cw_s[t][sub];
            const float cw[4] = {c4.x, c4.y, c4.z, c4.w};
            float f0 = 0.f, f1 = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) { f0 = fmaf(cw[i], f[i].x, f0); f1 = fmaf(cw[i], f[i].y, f1); }
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { f0 += __shfl_xor_sync(0xffffffffu, f0, o); f1 += __shfl_xor_sync(0xffffffffu, f1, o); }
            if (sub == 0 && e < n_entries) out[(int64_t)t * n_entries + e] = make_float2(f0, f1);
        }
    }
}
}  // namespace nsb

extern "C" int nsb_blend_tables(const nsb_field_params *params, const nsb_field_opts *opts, int32_t first_timestep,
                                int32_t n_timesteps, int64_t n_entries, void *out, void *stream) {
    if (!params || !opts || !out || !params->tables || !params->blend_codes) { set_error("nsb_blend_tables: null argument"); return 1; }
    if (first_timestep < 0 || n_timesteps < 1 || n_timesteps > kBlendMaxTimesteps || first_timestep > params->n_timesteps - n_timesteps) {
        set_error("nsb_blend_tables: timesteps [%d, %d + %d) out of range (n_timesteps %d, at most %d per call)", first_timestep,
                  first_timestep, n_timesteps, params->n_timesteps, kBlendMaxTimesteps);
        return 1;
    }
    if (n_entries <= 0) return 0;
    const int blocks = (int)std::min<int64_t>((n_entries + 31) / 32, (int64_t)num_sms() * 8);
    blend_tables_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4 *>(params->tables),
                                                                  params->blend_codes + (size_t)first_timestep * NSB_MEMBERS, *opts,
                                                                  reinterpret_cast<float2 *>(out), n_timesteps, n_entries);
    return check_launch("blend_tables_kernel");
}

// -------------------------------------------------------------------------------------------
// nsb_render_forward: host side of render_kernel_ws
// -------------------------------------------------------------------------------------------
namespace nsb {
// The render kernels run one CTA per SM, all resident: the grid barriers rely on it (the cooperative launch checks it).
template <int SAMPLER, bool FR, bool ST>
static int launch_render_tc_(const RenderKArgs &K, cudaStream_t st) {
    if (!tc_args_ok(K.F)) return 1;
    return launch_persistent<render_kernel_tc<SAMPLER, FR, ST>>(K, tc_smem_bytes<FR>(tc_code_bias_rows<FR>(K.F.P.n_timesteps)),
                                                                tc_smem_bytes<FR>(tc_code_bias_rows<FR>(kTcCodeBiasRows)),
                                                                num_sms(), &K.hdr->barrier, "render_kernel_tc", st);
}
template <int SAMPLER>
static int launch_render_tc(const RenderKArgs &K, cudaStream_t st) {
    if (!K.F.P.frame_table) return launch_render_tc_<SAMPLER, false, false>(K, st);
    return K.F.P.frame_stride ? launch_render_tc_<SAMPLER, true, true>(K, st) : launch_render_tc_<SAMPLER, true, false>(K, st);
}

template <bool D, int SAMPLER>
static int launch_render(const RenderKArgs &K, cudaStream_t st) {
    if constexpr (D)
        if (K.F.P.deform_packed_umma)       // every instantiation is its own draw of ptxas' allocation: the fixed march
            // runs the <4> binary (run-time sampler choice, fixed march as a call), given samples the <2> binary
            return SAMPLER == 0 ? launch_render_tc<4>(K, st) : launch_render_tc<2>(K, st);
    return launch_persistent<render_kernel_ws<D, SAMPLER>>(K, sizeof(SmemWS), sizeof(SmemWS), num_sms(), &K.hdr->barrier,
                                                           "render_kernel_ws", st);
}
}  // namespace nsb

extern "C" size_t nsb_render_workspace_bytes(int64_t n_rays) {
    return kRenderHdrBytes + kRenderPartials * sizeof(int64_t) + (size_t)std::max<int64_t>(n_rays, 1) * sizeof(int32_t) + 64;
}

namespace nsb {
template <int SAMPLER, bool FR>
static int launch_render_tc_lerp_(const RenderKArgs &K, cudaStream_t st) {
    if (!tc_args_ok(K.F)) return 1;
    return launch_persistent<render_kernel_tc_lerp<SAMPLER, FR, FR>>(K, tc_smem_bytes<FR>(tc_code_bias_rows<FR>(K.F.P.n_timesteps)),
                                                                     tc_smem_bytes<FR>(tc_code_bias_rows<FR>(kTcCodeBiasRows)),
                                                                     num_sms(), &K.hdr->barrier, "render_kernel_tc_lerp", st);
}
template <int SAMPLER>
static int launch_render_tc_lerp(const RenderKArgs &K, cudaStream_t st) {
    return K.F.P.frame_table ? launch_render_tc_lerp_<SAMPLER, true>(K, st) : launch_render_tc_lerp_<SAMPLER, false>(K, st);
}

// The two render entry points share their checks and argument set-up; `lerp` selects render_kernel_tc_lerp.
static int render_forward(const char *who, const bool lerp, const nsb_field_params *params, const nsb_field_opts *opts,
                          const nsb_render_args *ra, void *stream) {
    if (!params || !opts || !ra) { set_error("%s: null argument", who); return 1; }
    if (ra->n_rays <= 0) return 0;
    if (check_field_params(who, params)) return 1;
    const bool deform = opts->use_deformation != 0;
    if (!ra->origins || !ra->directions || !ra->t_starts || !ra->t_ends || !ra->ray_indices || !ra->sigma || !ra->rgb ||
        !ra->packed_info || !ra->out_rgb || !ra->out_acc || !ra->out_depth || !ra->workspace || (deform && !ra->offsets)) {
        set_error("%s: null buffer", who);
        return 1;
    }
    if (!params->tables || !params->field_packed || !params->blend_codes) { set_error("%s: tables/field_packed/blend_codes missing", who); return 1; }
    if (deform && (!params->deform_packed_tb || !params->deform_bias || !params->deform_code_bias)) {
        set_error("%s: deformation parameters missing", who);
        return 1;
    }
    if (ra->capacity <= 0) { set_error("%s: capacity <= 0", who); return 1; }
    if (ra->sampler == 0) {
        if (ra->n_per_ray <= 0 || ra->capacity < ra->n_rays * (int64_t)ra->n_per_ray) { set_error("%s: capacity < n_rays * n_per_ray", who); return 1; }
    } else if (ra->sampler == 1) {
        if (!ra->near_planes || !ra->far_planes || !ra->binaries || !ra->aabbs) { set_error("%s: occupancy sampler arguments", who); return 1; }
        if (ra->levels < 1 || ra->levels > 8) { set_error("%s: levels must be in [1,8]", who); return 1; }
    } else { set_error("%s: unknown sampler", who); return 1; }
    if (lerp) {
        // the linear kernels are render_kernel_tc with the deformation MLP on wgmma; a frame table must be the stack of
        // every timestep (one frame's table holds one timestep)
        if (!deform) { set_error("%s: linear time needs the deformation field (use_deformation)", who); return 1; }
        if (!params->deform_packed_umma) { set_error("%s: linear time needs the wgmma deformation weights (deform_packed_umma)", who); return 1; }
        if (params->frame_table && params->frame_stride < params->levels.offset[NSB_MAX_LEVELS - 1] + (int64_t)params->levels.entries[NSB_MAX_LEVELS - 1]) {
            set_error("%s: the frame table must be a timestep stack whose frame_stride covers every level's entries", who);
            return 1;
        }
    }
    uint8_t *ws = reinterpret_cast<uint8_t *>(ra->workspace);
    RenderKArgs K;
    memset(&K, 0, sizeof(K));
    K.hdr = reinterpret_cast<nsb_render_ws_header *>(ws);
    K.partials = reinterpret_cast<int64_t *>(ws + kRenderHdrBytes);
    int32_t *counts = reinterpret_cast<int32_t *>(ws + kRenderHdrBytes + kRenderPartials * sizeof(int64_t));
    K.F.P = *params; K.F.O = *opts;
    K.F.O.compute_rgb = 1;
    for (int k = 0; k < 3; ++k) K.F.aabb_size[k] = params->aabb[3 + k] - params->aabb[k];
    K.F.S.n_samples = 0;                 // device-side: sm.n_dyn
    K.F.S.origins = ra->origins; K.F.S.directions = ra->directions; K.F.S.ray_times = ra->ray_times;
    K.F.S.t_starts = ra->t_starts; K.F.S.t_ends = ra->t_ends; K.F.S.ray_indices = ra->ray_indices;
    K.F.out.sigma = ra->sigma; K.F.out.rgb = ra->rgb; K.F.out.offsets = deform ? ra->offsets : nullptr;
    K.M.n_rays = ra->n_rays; K.M.origins = ra->origins; K.M.directions = ra->directions;
    K.M.near_planes = ra->near_planes; K.M.far_planes = ra->far_planes; K.M.binaries = ra->binaries; K.M.aabbs = ra->aabbs;
    K.M.levels = ra->levels; K.M.res = ra->res; K.M.step = ra->step; K.M.cone_angle = ra->cone_angle;
    K.M.counts = counts; K.M.offsets = nullptr; K.M.t_starts = ra->t_starts; K.M.t_ends = ra->t_ends; K.M.ray_indices = ra->ray_indices;
    K.C.n_rays = ra->n_rays; K.C.n_samples = ra->capacity; K.C.packed_info = ra->packed_info; K.packed_info = ra->packed_info;
    K.C.t_starts = ra->t_starts; K.C.t_ends = ra->t_ends; K.C.sigma = ra->sigma; K.C.rgb = ra->rgb;
    K.C.offsets = deform ? ra->offsets : nullptr; K.C.training = ra->training;
    K.C.out_rgb = ra->out_rgb; K.C.out_acc = ra->out_acc; K.C.out_depth = ra->out_depth;
    K.C.out_deform = deform ? ra->out_deform : nullptr; K.C.out_weights = ra->weights;
    K.C.workspace = K.hdr->depth_range;
    K.sampler = ra->sampler; K.n_per_ray = ra->n_per_ray; K.near_plane = ra->near_plane; K.capacity = ra->capacity;
    cudaStream_t st = (cudaStream_t)stream;
    if (ra->sampler == 1) {
        // occupancy march as its own small cooperative launch (count | scan | fill, the count stays on the device), then
        // field + composite in one: with the marcher inside render_kernel_ws ptxas spilled 66-82 instructions in the
        // gather role of the field phase (tools/spill_report.py).
        const int rc = launch_march_occ_coop(K.M, K.packed_info, K.hdr, K.partials, K.capacity, ra->march_scratch, st);
        if (rc) return rc;
        if (lerp) return launch_render_tc_lerp<2>(K, st);
        return deform ? launch_render<true, 2>(K, st) : launch_render<false, 2>(K, st);
    }
    if (lerp) return launch_render_tc_lerp<4>(K, st);
    return deform ? launch_render<true, 0>(K, st) : launch_render<false, 0>(K, st);
}
}  // namespace nsb

extern "C" int nsb_render_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_render_args *ra, void *stream) {
    return render_forward("nsb_render_forward", false, params, opts, ra, stream);
}

extern "C" int nsb_render_forward_interp(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_render_args *ra,
                                         void *stream) {
    return render_forward("nsb_render_forward_interp", true, params, opts, ra, stream);
}
