// Surface normals of the density field: nerfstudio's Field.get_normals (n = -normalize(d h0 / d x), h0 = mlp_base output 0
// before trunc_exp, x = the normalised hash-input position after the in-box selector) and NormalsRenderer(normalize=True)
// over packed samples.  A separate pass over samples the field / render kernels already produced: it re-gathers the same
// tables (blended frame table / timestep stack, or the 128 B lines with table or per-sample blend codes) and leaves the
// fused kernels alone.
//
// normals_kernel: persistent, one warp per sample.  Lane = (level lane >> 1, z half lane & 1) as in the frame gather role:
// the lane's 4 corners give the level's two features and their spatial derivatives (trilinear weight derivative times
// the level scale, the math of the position gradient in nsb_backward.cu); the two z halves meet in one shuffle, after
// which lane j holds feature j and d feat_j / d x.  mlp_base layer 0 runs in fp32 FMAs from shared memory for the ReLU
// mask, d h0 / d feat = W0^T (W1[0] . mask), and a warp sum contracts it with d feat / d x.
// normals_observation_kernel (observation_space): one thread per sample turns the unit canonical normal n and
// d = J^T D^-1 n (nsb_deform_vjp.cu) into n_obs = normalize(grad_scale * s * (n + d)); n already carries the minus sign.
// normals_composite_kernel: one warp per ray sums w_i * n_i over its packed segment in a fixed order (no atomics).
#include <algorithm>

#include "nsb_gather.cuh"

namespace nsb {
namespace {

constexpr int kNrmWarps = 8;
constexpr int kW0Pitch = 65;   // [input k][hidden n] rows of 65: row reads (fixed k) and column reads (fixed n) are conflict-free

struct NormalsKArgs {
    nsb_field_params P;
    nsb_field_opts O;
    nsb_samples S;
    nsb_normals_args N;
    float aabb_size[3];
};

struct SmemNormals {
    float w0[32 * kW0Pitch];          // mlp_base layer 0 (fp16 values), w0[k * 65 + n] = W0[n][k]
    float w1[64];                     // mlp_base layer 1, output row 0 (h0)
    float cw[kNrmWarps][NSB_MEMBERS]; // line gather: the sample's fp16-rounded member weights, one row per warp
};

// Element i of a matrix packed by python pack_mma_b (order [k-tile][n-tile pair][g][q][ntsel][hi][e]) with `pairs`
// n-tile pairs per k-tile: its (output n, input k).
__device__ __forceinline__ void mma_b_coords(int i, int pairs, int &n, int &k) {
    const int e = i & 1, hi = (i >> 1) & 1, ntsel = (i >> 2) & 1, q = (i >> 3) & 3, g = (i >> 5) & 7, rest = i >> 8;
    n = (rest % pairs) * 16 + ntsel * 8 + g;
    k = (rest / pairs) * 16 + hi * 8 + 2 * q + e;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <bool FRAME>
__global__ void __launch_bounds__(kNrmWarps * 32) normals_kernel(const __grid_constant__ NormalsKArgs K) {
    __shared__ SmemNormals sm;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    {   // mlp_base from the packed fp16 field weights (layer 0: 2048 halfs, 4 pairs; layer 1: 1024 halfs, 1 pair)
        const __half *fp = reinterpret_cast<const __half *>(K.P.field_packed);
        for (int i = tid; i < 2048; i += kNrmWarps * 32) {
            int n, k;
            mma_b_coords(i, 4, n, k);
            sm.w0[k * kW0Pitch + n] = __half2float(fp[i]);
        }
        for (int i = tid; i < 1024; i += kNrmWarps * 32) {
            int n, k;
            mma_b_coords(i, 1, n, k);
            if (n == 0) sm.w1[k] = __half2float(fp[2048 + i]);
        }
    }
    __syncthreads();
    const int64_t n = K.S.n_samples_dev ? min(*K.S.n_samples_dev, K.S.n_samples) : K.S.n_samples;
    const int lvl = lane >> 1;
    const uint32_t dz = lane & 1;
    const float scale = K.P.levels.scale[lvl];
    const uint32_t res = K.P.levels.res[lvl], ent = K.P.levels.entries[lvl], off = K.P.levels.offset[lvl];
    const bool hashed = K.P.levels.hashed[lvl] != 0;
    const float amin0 = K.P.aabb[0], amin1 = K.P.aabb[1], amin2 = K.P.aabb[2];
    float *const cw = sm.cw[warp];
    for (int64_t s = (int64_t)blockIdx.x * kNrmWarps + warp; s < n; s += (int64_t)gridDim.x * kNrmWarps) {
        // the sample's position and timestep, formed exactly as the field kernels form them
        float px, py, pz, tt = 0.f;
        if (K.S.origins) {
            const int64_t ri = K.S.ray_indices[s];
            const float mid = __fadd_rn(K.S.t_starts[s], K.S.t_ends[s]);
            const float ddx = K.S.directions[3 * ri + 0], ddy = K.S.directions[3 * ri + 1], ddz = K.S.directions[3 * ri + 2];
            px = ray_midpoint(K.S.origins[3 * ri + 0], ddx, mid);
            py = ray_midpoint(K.S.origins[3 * ri + 1], ddy, mid);
            pz = ray_midpoint(K.S.origins[3 * ri + 2], ddz, mid);
            if (K.S.ray_times) tt = K.S.ray_times[ri];
        } else {
            px = K.S.positions[3 * s + 0]; py = K.S.positions[3 * s + 1]; pz = K.S.positions[3 * s + 2];
            if (K.S.sample_times) tt = K.S.sample_times[s];
        }
        const int tsi = sample_timestep(tt, K.P.n_timesteps);
        if (K.N.offsets) {      // normalised offsets added to WORLD coordinates (the reference's quirk, as the field kernels)
            px = __fadd_rn(px, K.N.offsets[3 * s + 0]);
            py = __fadd_rn(py, K.N.offsets[3 * s + 1]);
            pz = __fadd_rn(pz, K.N.offsets[3 * s + 2]);
        }
        float x = box_coord(px, amin0, K.aabb_size[0]);
        float y = box_coord(py, amin1, K.aabb_size[1]);
        float z = box_coord(pz, amin2, K.aabb_size[2]);
        // outside the box x = 0: the normal is the gradient at the box origin (the selector multiplies the position,
        // it does not mask the gradient)
        if (!((x > 0.f) && (x < 1.f) && (y > 0.f) && (y < 1.f) && (z > 0.f) && (z < 1.f))) x = y = z = 0.f;
        if (!FRAME) {   // member weights, rounded to fp16 like the forward's blend operand (make_blend_b)
            const float *code_row = K.S.sample_blend_codes ? K.S.sample_blend_codes + s * NSB_MEMBERS
                                                           : K.P.blend_codes + (size_t)tsi * NSB_MEMBERS;
            cw[lane] = __half2float(__float2half_rn(fmaf(code_row[lane], K.O.cw_scale[lane], K.O.cw_bias[lane])));
            __syncwarp();
        }
        // this lane's 4 corners of level lvl: features (f0, f1) and d / d frac of each
        const float qx = fmaf(scale, x, 0.5f), qy = fmaf(scale, y, 0.5f), qz = fmaf(scale, z, 0.5f);
        const float flx = floorf(qx), fly = floorf(qy), flz = floorf(qz);
        const float fx = qx - flx, fy = qy - fly, fz = qz - flz;
        const uint32_t cx0 = (uint32_t)(int)flx, cy0 = (uint32_t)(int)fly, cz = (uint32_t)(int)flz + dz;
        const float wz = dz ? fz : 1.0f - fz;
        const float2 *ft = nullptr;
        if (FRAME) {    // stack: timestep * frame_stride + entry < 2^32 (checked on the host)
            ft = reinterpret_cast<const float2 *>(K.P.frame_table) + off;
            ft += (uint32_t)tsi * (uint32_t)K.P.frame_stride;
        }
        float f0 = 0.f, f1 = 0.f, g0x = 0.f, g0y = 0.f, g0z = 0.f, g1x = 0.f, g1y = 0.f, g1z = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t dx = c & 1, dy = c >> 1;
            const uint32_t idx = grid_index(hashed, res, ent, cx0 + dx, cy0 + dy, cz);
            float2 v;
            if (FRAME) {
                v = __ldg(ft + idx);
            } else {
                const uint4 *ln = reinterpret_cast<const uint4 *>(reinterpret_cast<const uint8_t *>(K.P.tables) + (size_t)(off + idx) * 128);
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {   // members 4j .. 4j + 3
                    const uint4 u = __ldg(ln + j);
                    const float4 w4 = *reinterpret_cast<const float4 *>(cw + 4 * j);
                    float2 m = unpack_h2(u.x); a0 = fmaf(w4.x, m.x, a0); a1 = fmaf(w4.x, m.y, a1);
                    m = unpack_h2(u.y); a0 = fmaf(w4.y, m.x, a0); a1 = fmaf(w4.y, m.y, a1);
                    m = unpack_h2(u.z); a0 = fmaf(w4.z, m.x, a0); a1 = fmaf(w4.z, m.y, a1);
                    m = unpack_h2(u.w); a0 = fmaf(w4.w, m.x, a0); a1 = fmaf(w4.w, m.y, a1);
                }
                v = make_float2(a0, a1);
            }
            const float wx = dx ? fx : 1.0f - fx, wy = dy ? fy : 1.0f - fy;
            const float w = (wx * wy) * wz;
            // d w / d frac_d: +- the product of the other two factors
            const float ex = (dx ? wy : -wy) * wz, ey = (dy ? wx : -wx) * wz, ez = dz ? wx * wy : -(wx * wy);
            f0 = fmaf(w, v.x, f0); f1 = fmaf(w, v.y, f1);
            g0x = fmaf(ex, v.x, g0x); g0y = fmaf(ey, v.x, g0y); g0z = fmaf(ez, v.x, g0z);
            g1x = fmaf(ex, v.y, g1x); g1y = fmaf(ey, v.y, g1y); g1z = fmaf(ez, v.y, g1z);
        }
        if (!FRAME) __syncwarp();   // every lane has read cw before the next sample rewrites it
        f0 += __shfl_xor_sync(0xffffffffu, f0, 1); f1 += __shfl_xor_sync(0xffffffffu, f1, 1);
        g0x += __shfl_xor_sync(0xffffffffu, g0x, 1); g0y += __shfl_xor_sync(0xffffffffu, g0y, 1);
        g0z += __shfl_xor_sync(0xffffffffu, g0z, 1); g1x += __shfl_xor_sync(0xffffffffu, g1x, 1);
        g1y += __shfl_xor_sync(0xffffffffu, g1y, 1); g1z += __shfl_xor_sync(0xffffffffu, g1z, 1);
        // lane j = 2 * level + feat: feature j and d feat_j / d x (d frac / d x = scale)
        const bool odd = lane & 1;
        const float feat = odd ? f1 : f0;
        const float dfx = scale * (odd ? g1x : g0x), dfy = scale * (odd ? g1y : g0y), dfz = scale * (odd ? g1z : g0z);
        // mlp_base layer 0 on the fp16-rounded features (the MLP's input operand): hidden units lane and lane + 32
        const float fh = __half2float(__float2half_rn(feat));
        float h_lo = 0.f, h_hi = 0.f;
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const float fj = __shfl_sync(0xffffffffu, fh, j);
            h_lo = fmaf(sm.w0[j * kW0Pitch + lane], fj, h_lo);
            h_hi = fmaf(sm.w0[j * kW0Pitch + 32 + lane], fj, h_hi);
        }
        const float m_lo = h_lo > 0.f ? sm.w1[lane] : 0.f, m_hi = h_hi > 0.f ? sm.w1[32 + lane] : 0.f;
        // d h0 / d feat_lane = sum_i W1[0][i] mask_i W0[i][lane]
        float dh = 0.f;
#pragma unroll 8
        for (int i = 0; i < 32; ++i) {
            dh = fmaf(__shfl_sync(0xffffffffu, m_lo, i), sm.w0[lane * kW0Pitch + i], dh);
            dh = fmaf(__shfl_sync(0xffffffffu, m_hi, i), sm.w0[lane * kW0Pitch + 32 + i], dh);
        }
        const float gx = warp_sum(dh * dfx) * K.N.grad_scale[0];
        const float gy = warp_sum(dh * dfy) * K.N.grad_scale[1];
        const float gz = warp_sum(dh * dfz) * K.N.grad_scale[2];
        // -F.normalize(g): g / max(|g|, 1e-12)
        const float den = fmaxf(sqrtf(gx * gx + gy * gy + gz * gz), 1e-12f);
        if (lane < 3) K.N.normals[3 * s + lane] = -(lane == 0 ? gx : (lane == 1 ? gy : gz)) / den;
    }
}

// Observation-space normals from the canonical ones: the chain rule through x = s * (p_n + D^-1 offset(p_n)).  The warped
// position and its in-box selector s are formed as normals_kernel forms them.
__global__ void __launch_bounds__(256) normals_observation_kernel(const __grid_constant__ NormalsKArgs K) {
    const int64_t n = K.S.n_samples_dev ? min(*K.S.n_samples_dev, K.S.n_samples) : K.S.n_samples;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (int64_t)gridDim.x * blockDim.x) {
        float px, py, pz;
        if (K.S.origins) {
            const int64_t ri = K.S.ray_indices[s];
            const float mid = __fadd_rn(K.S.t_starts[s], K.S.t_ends[s]);
            px = ray_midpoint(K.S.origins[3 * ri + 0], K.S.directions[3 * ri + 0], mid);
            py = ray_midpoint(K.S.origins[3 * ri + 1], K.S.directions[3 * ri + 1], mid);
            pz = ray_midpoint(K.S.origins[3 * ri + 2], K.S.directions[3 * ri + 2], mid);
        } else {
            px = K.S.positions[3 * s + 0]; py = K.S.positions[3 * s + 1]; pz = K.S.positions[3 * s + 2];
        }
        px = __fadd_rn(px, K.N.offsets[3 * s + 0]);
        py = __fadd_rn(py, K.N.offsets[3 * s + 1]);
        pz = __fadd_rn(pz, K.N.offsets[3 * s + 2]);
        const float x = box_coord(px, K.P.aabb[0], K.aabb_size[0]);
        const float y = box_coord(py, K.P.aabb[1], K.aabb_size[1]);
        const float z = box_coord(pz, K.P.aabb[2], K.aabb_size[2]);
        const bool sel = (x > 0.f) && (x < 1.f) && (y > 0.f) && (y < 1.f) && (z > 0.f) && (z < 1.f);
        float v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            v[k] = sel ? K.N.grad_scale[k] * (K.N.normals[3 * s + k] + K.N.vjp_scratch[3 * s + k]) : 0.f;
        const float den = fmaxf(sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]), 1e-12f);
#pragma unroll
        for (int k = 0; k < 3; ++k) K.N.normals[3 * s + k] = v[k] / den;
    }
}

// NormalsRenderer(normalize=True): N = v / (|v| + 1e-10), v = sum_i w_i n_i over the ray's samples.  Each lane sums a fixed
// stride of the segment, then a fixed butterfly: the result is the same bits on every run.
__global__ void __launch_bounds__(256) normals_composite_kernel(const __grid_constant__ NormalsKArgs K) {
    const int lane = threadIdx.x & 31;
    const int64_t n = K.S.n_samples_dev ? min(*K.S.n_samples_dev, K.S.n_samples) : K.S.n_samples;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < K.N.n_rays; r += warps) {
        const int64_t start = K.N.packed_info[2 * r], end = min(start + K.N.packed_info[2 * r + 1], n);
        float ax = 0.f, ay = 0.f, az = 0.f;
        for (int64_t i = start + lane; i < end; i += 32) {
            const float w = K.N.weights[i];
            ax = fmaf(w, K.N.normals[3 * i + 0], ax);
            ay = fmaf(w, K.N.normals[3 * i + 1], ay);
            az = fmaf(w, K.N.normals[3 * i + 2], az);
        }
        ax = warp_sum(ax); ay = warp_sum(ay); az = warp_sum(az);
        const float den = sqrtf(ax * ax + ay * ay + az * az) + 1e-10f;
        if (lane < 3) K.N.out_normals[3 * r + lane] = (lane == 0 ? ax : (lane == 1 ? ay : az)) / den;
    }
}

}  // namespace
}  // namespace nsb

using namespace nsb;

extern "C" int nsb_normals_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                                   const nsb_normals_args *args, void *stream) {
    if (!params || !opts || !samples || !args) { set_error("nsb_normals_forward: null argument"); return 1; }
    if (!args->normals) {
        if (args->out_normals) { set_error("nsb_normals_forward: out_normals needs the per-sample normals buffer"); return 1; }
        return 0;
    }
    if (args->out_normals && (!args->packed_info || !args->weights || args->n_rays < 0)) {
        set_error("nsb_normals_forward: out_normals needs packed_info, n_rays and weights");
        return 1;
    }
    if (check_field_params("nsb_normals_forward", params) || check_samples("nsb_normals_forward", samples)) return 1;
    if (!params->field_packed) { set_error("nsb_normals_forward: field_packed missing"); return 1; }
    const bool frame = params->frame_table != nullptr;
    if (!frame && (!params->tables || (!params->blend_codes && !samples->sample_blend_codes))) {
        set_error("nsb_normals_forward: tables / blend codes missing");
        return 1;
    }
    const bool observation = args->observation_space != 0;
    if (observation && (!opts->use_deformation || !args->offsets || !args->vjp_scratch)) {
        set_error("nsb_normals_forward: observation_space needs use_deformation, offsets and vjp_scratch");
        return 1;
    }
    if (samples->n_samples <= 0) return 0;
    NormalsKArgs K;
    K.P = *params; K.O = *opts; K.S = *samples; K.N = *args;
    for (int k = 0; k < 3; ++k) K.aabb_size[k] = params->aabb[3 + k] - params->aabb[k];
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = (int)std::min<int64_t>((samples->n_samples + kNrmWarps - 1) / kNrmWarps, (int64_t)num_sms() * 8);
    if (observation)        // the canonical pass leaves -g / |g| of the normalised hash input; grad_scale applies at the end
        for (int k = 0; k < 3; ++k) K.N.grad_scale[k] = 1.0f;
    if (frame) normals_kernel<true><<<grid, kNrmWarps * 32, 0, st>>>(K);
    else normals_kernel<false><<<grid, kNrmWarps * 32, 0, st>>>(K);
    int rc = check_launch("normals_kernel");
    if (!rc && observation) {
        nsb_deform_vjp_args V;
        V.deform_packed_t = args->deform_packed_t; V.deform_packed_pe_t = args->deform_packed_pe_t;
        V.u = args->normals; V.loss_scale = args->loss_scale; V.d_pn = args->vjp_scratch;
        const float inv_extent[3] = {1.0f / K.aabb_size[0], 1.0f / K.aabb_size[1], 1.0f / K.aabb_size[2]};
        rc = launch_deform_input_grad("nsb_normals_forward", params, opts, samples, &V, inv_extent, st);
        if (rc) return rc;
        for (int k = 0; k < 3; ++k) K.N.grad_scale[k] = args->grad_scale[k];
        const int ogrid = (int)std::min<int64_t>((samples->n_samples + 255) / 256, (int64_t)num_sms() * 8);
        normals_observation_kernel<<<ogrid, 256, 0, st>>>(K);
        rc = check_launch("normals_observation_kernel");
    }
    if (rc || !args->out_normals || args->n_rays == 0) return rc;
    const int rgrid = (int)std::min<int64_t>((args->n_rays + 7) / 8, (int64_t)num_sms() * 8);
    normals_composite_kernel<<<rgrid, 256, 0, st>>>(K);
    return check_launch("normals_composite_kernel");
}
