// Fused optimiser step for the hash tables: rank-1 gradient expansion + Adam + fp16 shadow refresh in one pass.
// HBM-bound streaming kernel: per table line it reads p, m, v (3 x 256 B) and the scatter workspace (8 B per slot),
// writes p, m, v (3 x 256 B) and the fp16 line (128 B): 1.66 KB + 8 B x n_slots per line, 10.5 + 1.2 GB for the
// 6.3 M-line / 24-timestep configuration.  See include/nsb.h (nsb_table_adam_step) for what it replaces.
#include "nsb_common.cuh"

namespace nsb {

constexpr int kOptWarps = 4;        // warps per block
constexpr int kOptLines = 32;       // table lines per warp iteration
constexpr int kOptMaxSlots = 32;

struct AdamK {
    nsb_table_adam_args a;
};

// One warp owns kOptLines consecutive lines per iteration.
//   phase 1: for every slot, the 32 lanes read the slot's 2-vectors of the 32 lines (one coalesced 256 B read) into the
//            warp's shared-memory panel gs[slot][line].
//   phase 2: per line, lane = ensemble member: g[f] = sum_slots cw[slot][member] * gs[slot][line][f] (panel reads are
//            broadcasts), then the Adam update of (line, member, f = 0, 1): every array access is one coalesced
//            256 B (fp32) or 128 B (fp16) row per warp.
template <bool ADAM>
__global__ void __launch_bounds__(kOptWarps * 32) table_step_kernel(const __grid_constant__ AdamK K, float *d_tables) {
    __shared__ float2 gs[kOptWarps][kOptMaxSlots][kOptLines];
    const nsb_table_adam_args &a = K.a;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n_slots = a.g_rank1 ? a.n_slots : 0;
    float cw[kOptMaxSlots];
#pragma unroll
    for (int sl = 0; sl < kOptMaxSlots; ++sl) cw[sl] = sl < n_slots ? a.cw_slots[sl * NSB_MEMBERS + lane] : 0.f;
    const int64_t E = a.total_entries;
    const int64_t n_blocks = (E + kOptLines - 1) / kOptLines;
    const float w1 = a.one_minus_beta1, w2 = a.one_minus_beta2;
    const float step_size = a.step_size, bc2_sqrt = a.bias_correction2_sqrt;
    for (int64_t blk = (int64_t)blockIdx.x * kOptWarps + warp; blk < n_blocks; blk += (int64_t)gridDim.x * kOptWarps) {
        const int64_t e0 = blk * kOptLines;
        if (ADAM) {   // pull the NEXT block's p / m / v lines (3 x 8 KB) into L2 while this one is processed
            const int64_t nb = blk + (int64_t)gridDim.x * kOptWarps;
            if (nb < n_blocks) {
                const size_t o = (size_t)nb * kOptLines * NSB_MEMBERS * 2 + (size_t)lane * 64;   // lane -> 256 B line-pair
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a.tables + o + h * 32));
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a.exp_avg + o + h * 32));
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a.exp_avg_sq + o + h * 32));
                }
            }
        }
        unsigned any_slot = 0;   // bit sl: some line of this block has a non-zero vector in slot sl (warp-uniform)
        for (int s0 = 0; s0 < n_slots; s0 += 8) {      // 8 slot rows in flight (a ballot per load serialises them)
            float2 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                v[u] = make_float2(0.f, 0.f);
                if (s0 + u < n_slots && e0 + lane < E)
                    v[u] = __ldg(reinterpret_cast<const float2 *>(a.g_rank1 + ((size_t)(s0 + u) * E + e0 + lane) * 2));
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (s0 + u >= n_slots) break;
                gs[warp][s0 + u][lane] = v[u];
                if (__ballot_sync(0xffffffffu, v[u].x != 0.f || v[u].y != 0.f)) any_slot |= 1u << (s0 + u);
            }
        }
        __syncwarp();
        const int lines = (int)min((int64_t)kOptLines, E - e0);
        constexpr int U = 4;    // lines in flight per warp: 12 x 256 B loads outstanding (one line at a time leaves HBM idle)
        for (int j0 = 0; j0 < lines; j0 += U) {
            float2 p[U], m[U], v[U], d[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const bool ok = j0 + u < lines;
                const size_t o = ((size_t)(e0 + (ok ? j0 + u : 0)) * NSB_MEMBERS + lane) * 2;
                d[u] = make_float2(0.f, 0.f);
                if (ADAM) {
                    p[u] = *reinterpret_cast<const float2 *>(a.tables + o);
                    m[u] = *reinterpret_cast<const float2 *>(a.exp_avg + o);
                    v[u] = *reinterpret_cast<const float2 *>(a.exp_avg_sq + o);
                }
                if (a.grad) d[u] = __ldg(reinterpret_cast<const float2 *>(a.grad + o));
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int j = j0 + u;
                if (j >= lines) continue;
                const size_t o = ((size_t)(e0 + j) * NSB_MEMBERS + lane) * 2;
                float g0 = 0.f, g1 = 0.f;
#pragma unroll
                for (int sl = 0; sl < kOptMaxSlots; ++sl) {
                    if (!((any_slot >> sl) & 1)) continue;
                    const float2 gv = gs[warp][sl][j];
                    g0 = fmaf(cw[sl], gv.x, g0);
                    g1 = fmaf(cw[sl], gv.y, g1);
                }
                g0 = (g0 + d[u].x) * a.grad_scale;
                g1 = (g1 + d[u].y) * a.grad_scale;
                if (!ADAM) {
                    if (any_slot) {
                        float2 *dst = reinterpret_cast<float2 *>(d_tables + o);
                        float2 cur = *dst;
                        cur.x += g0; cur.y += g1;
                        *dst = cur;
                    }
                    continue;
                }
                float2 pp = p[u], mm = m[u], vv = v[u];
                if (a.weight_decay != 0.f) { g0 = fmaf(a.weight_decay, pp.x, g0); g1 = fmaf(a.weight_decay, pp.y, g1); }
                // torch.optim.Adam on CUDA (_multi_tensor_adam), operation by operation and with its roundings, so that
                // the step is bit-identical to torch's for the same gradient:
                //   exp_avg.lerp_(grad, 1 - beta1)                 m + w1 * (g - m), one fma
                //   exp_avg_sq.mul_(beta2).addcmul_(g, g, 1 - beta2)   v * beta2 rounded, then v + w2 * (g * g), one fma
                //   denom = exp_avg_sq.sqrt() / sqrt(bc2) + eps;  param.addcdiv_(exp_avg, denom, -lr / bc1)   one fma
                mm.x = fmaf(w1, g0 - mm.x, mm.x); mm.y = fmaf(w1, g1 - mm.y, mm.y);
                vv.x = fmaf(w2, __fmul_rn(g0, g0), __fmul_rn(vv.x, a.beta2));
                vv.y = fmaf(w2, __fmul_rn(g1, g1), __fmul_rn(vv.y, a.beta2));
                pp.x = fmaf(-step_size, __fdiv_rn(mm.x, __fadd_rn(__fdiv_rn(__fsqrt_rn(vv.x), bc2_sqrt), a.eps)), pp.x);
                pp.y = fmaf(-step_size, __fdiv_rn(mm.y, __fadd_rn(__fdiv_rn(__fsqrt_rn(vv.y), bc2_sqrt), a.eps)), pp.y);
                *reinterpret_cast<float2 *>(a.tables + o) = pp;
                *reinterpret_cast<float2 *>(a.exp_avg + o) = mm;
                *reinterpret_cast<float2 *>(a.exp_avg_sq + o) = vv;
                if (a.tables_half)
                    reinterpret_cast<__half2 *>(a.tables_half)[(size_t)(e0 + j) * NSB_MEMBERS + lane] = __floats2half2_rn(pp.x, pp.y);
            }
        }
        __syncwarp();
    }
}

static int opt_grid() {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
    return sms * 8;   // 32 KB of shared memory per block: 7 blocks fit, 8 per SM keeps every SM at its residency limit
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_table_adam_step(const nsb_table_adam_args *args, void *stream) {
    if (!args || !args->tables || !args->exp_avg || !args->exp_avg_sq) { set_error("nsb_table_adam_step: null argument"); return 1; }
    if (args->total_entries <= 0) return 0;
    if (!args->grad && !args->g_rank1) { set_error("nsb_table_adam_step: neither a dense gradient nor a rank-1 workspace"); return 1; }
    if (args->g_rank1 && (!args->cw_slots || args->n_slots < 1 || args->n_slots > kOptMaxSlots)) {
        set_error("nsb_table_adam_step: rank-1 workspace needs cw_slots and 1 <= n_slots <= 32");
        return 1;
    }
    if (!(args->bias_correction1 > 0.f) || !(args->bias_correction2 > 0.f) || !(args->bias_correction2_sqrt > 0.f)) {
        set_error("nsb_table_adam_step: bias corrections must be > 0 (step >= 1)");
        return 1;
    }
    AdamK K;
    K.a = *args;
    table_step_kernel<true><<<opt_grid(), kOptWarps * 32, 0, (cudaStream_t)stream>>>(K, nullptr);
    return check_launch("table_step_kernel<adam>");
}

extern "C" int nsb_rank1_expand(const float *g_rank1, const float *cw_slots, int32_t n_slots, int64_t total_entries,
                                float grad_scale, float *d_tables, void *stream) {
    if (!g_rank1 || !cw_slots || !d_tables) { set_error("nsb_rank1_expand: null argument"); return 1; }
    if (n_slots < 1 || n_slots > kOptMaxSlots) { set_error("nsb_rank1_expand: 1 <= n_slots <= 32"); return 1; }
    if (total_entries <= 0) return 0;
    AdamK K = {};
    K.a.total_entries = total_entries;
    K.a.g_rank1 = g_rank1; K.a.cw_slots = cw_slots; K.a.n_slots = n_slots; K.a.grad_scale = grad_scale;
    K.a.beta1 = K.a.beta2 = 0.f; K.a.bias_correction1 = K.a.bias_correction2 = 1.f; K.a.lr = 0.f;
    table_step_kernel<false><<<opt_grid(), kOptWarps * 32, 0, (cudaStream_t)stream>>>(K, d_tables);
    return check_launch("table_step_kernel<expand>");
}
