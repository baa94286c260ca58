// Hash-ensemble gather device code (shared by the forward kernels and the table-gradient kernel).
#pragma once
#include "nsb_common.cuh"

namespace nsb {

// -------------------------------------------------------------------------------------------
// hash-ensemble gather + blend for ONE sample by a full warp.  lane = cg*8 + mg:
//   mg = member group (members 4mg..4mg+3 = 16 B of the 128 B line), cg = corner group
//   (dx = cg&1, dy = cg>>1; the lane handles dz = 0 and dz = 1).  Returns feature `lane`
//   (= level*2 + feat) summed over members and corners.
// tcnn semantics (grid.h): pos = fmaf(scale,x,0.5); floor; w = prod(dim? frac : 1-frac);
// dense index x + y*res + z*res^2 (mod entries) or (x ^ y*2654435761 ^ z*805459861) mod 2^log2T.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float butterfly(float lo_idx, float hi_idx, int bit, int lane) {
    const bool up = (lane >> bit) & 1;
    float send = up ? lo_idx : hi_idx;
    float keep = up ? hi_idx : lo_idx;
    return keep + __shfl_xor_sync(0xffffffffu, send, 1 << bit);
}

template <int LB>  // levels per load batch (2*LB LDG.128 in flight per lane)
__device__ __forceinline__ float gather_blend(const nsb_field_params &P, float x, float y, float z,
                                              const float (&cw)[4], int lane) {
    const int mg = lane & 7, cg = lane >> 3;
    const uint32_t dx = cg & 1, dy = cg >> 1;
    const uint8_t *tab = reinterpret_cast<const uint8_t *>(P.tables) + mg * 16;
    float s1 = 0.f, s2 = 0.f, s3 = 0.f, s4 = 0.f, result = 0.f;
#pragma unroll
    for (int lb = 0; lb < NSB_MAX_LEVELS; lb += LB) {
        uint4 v[LB][2];
        float w[LB][2];
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int l = lb + i;
            const float scale = P.levels.scale[l];
            const uint32_t res = P.levels.res[l], ent = P.levels.entries[l], off = P.levels.offset[l];
            float px = fmaf(scale, x, 0.5f), py = fmaf(scale, y, 0.5f), pz = fmaf(scale, z, 0.5f);
            float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
            float fx = px - flx, fy = py - fly, fz = pz - flz;
            uint32_t cx = (uint32_t)(int)flx + dx, cy = (uint32_t)(int)fly + dy, cz = (uint32_t)(int)flz;
            float wxy = (dx ? fx : 1.0f - fx) * (dy ? fy : 1.0f - fy);
            w[i][0] = wxy * (1.0f - fz);
            w[i][1] = wxy * fz;
            uint32_t i0, i1;
            if (P.levels.hashed[l]) {
                // hashed levels always have entries = 2^log2_hashmap_size (checked on the host)
                uint32_t hxy = cx ^ (cy * kPrimeY);
                uint32_t hz = cz * kPrimeZ;
                i0 = (hxy ^ hz) & (ent - 1);
                i1 = (hxy ^ (hz + kPrimeZ)) & (ent - 1);
            } else {
                // index < 2*entries for corner coords <= res, so `% entries` is one conditional subtract
                i0 = cx + cy * res + cz * res * res;
                i1 = i0 + res * res;
                i0 = i0 >= ent ? i0 - ent : i0;
                i1 = i1 >= ent ? i1 - ent : i1;
            }
            v[i][0] = __ldg(reinterpret_cast<const uint4 *>(tab + (size_t)(off + i0) * 128));
            v[i][1] = __ldg(reinterpret_cast<const uint4 *>(tab + (size_t)(off + i1) * 128));
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int l = lb + i;
            float p0 = 0.f, p1 = 0.f;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                float2 m0 = unpack_h2(v[i][c].x), m1 = unpack_h2(v[i][c].y), m2 = unpack_h2(v[i][c].z),
                       m3 = unpack_h2(v[i][c].w);
                float in0 = cw[0] * m0.x + cw[1] * m1.x + cw[2] * m2.x + cw[3] * m3.x;
                float in1 = cw[0] * m0.y + cw[1] * m1.y + cw[2] * m2.y + cw[3] * m3.y;
                p0 = fmaf(w[i][c], in0, p0);
                p1 = fmaf(w[i][c], in1, p1);
            }
            // transposing butterfly: after level l the partial sums are merged like a binary counter
            float r = butterfly(p0, p1, 0, lane);
            if ((l & 1) == 0) { s1 = r; continue; }
            r = butterfly(s1, r, 1, lane);
            if ((l & 2) == 0) { s2 = r; continue; }
            r = butterfly(s2, r, 2, lane);
            if ((l & 4) == 0) { s3 = r; continue; }
            r = butterfly(s3, r, 3, lane);
            if ((l & 8) == 0) { s4 = r; continue; }
            result = butterfly(s4, r, 4, lane);
        }
    }
    return result;
}

// -------------------------------------------------------------------------------------------
// Tensor-core variant of the gather: the sum over the 32 ensemble members IS a dense contraction
//   out[line, f] = sum_m V[line, m, f] * cw[m]          (line = one (level, corner) table entry)
// so it runs as mma.sync m16n8k16 with A = 16 table lines x 16 halfs straight from the LDG
// registers (no conversion instructions), B = the sample's blend weights (fp16, like the
// reference: hash_ensemble.py:155 casts the code to half), fp32 accumulate.
//   m-tile t: rows 0-7 = level 2t corners 0-7, rows 8-15 = level 2t+1 corners 0-7.
//   lane (g,q) owns corner g of every level and loads bytes [32q,32q+32) of its two lines (ldg256: the 4 lanes
//   of a quad cover a whole 128 B line);
//   k-step s uses words s and 4+s, i.e. k=2q,2q+1 <-> member 8q+s (f0,f1) and k=2q+8,2q+9 <->
//   member 8q+4+s.  B[k][n] = cw[member(k)] * (feat(k)==n), n<2.
//   C (lanes q==0): c0,c1 = (level 2t, corner g, f0/f1); c2,c3 = (level 2t+1, corner g, f0/f1).
// Epilogue: times the lane's trilinear corner weight, then a 28-shuffle transposing butterfly
// over the corner lanes.  Returns feature `lane` (= level*2+feat) in every lane.
// -------------------------------------------------------------------------------------------
struct BlendB {
    uint32_t lo[4], hi[4];  // B fragments of the 4 k-steps (b0, b1)
};

__device__ __forceinline__ BlendB make_blend_b(const nsb_field_opts &O, const float *code_row, int lane) {
    const int g = lane >> 2, q = lane & 3;
    BlendB B;
    const float4 c0 = __ldg(reinterpret_cast<const float4 *>(code_row) + 2 * q);
    const float4 c1 = __ldg(reinterpret_cast<const float4 *>(code_row) + 2 * q + 1);
    const float lo[4] = {c0.x, c0.y, c0.z, c0.w}, hi[4] = {c1.x, c1.y, c1.z, c1.w};
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const float a = fmaf(lo[s], O.cw_scale[8 * q + s], O.cw_bias[8 * q + s]);
        const float b = fmaf(hi[s], O.cw_scale[8 * q + 4 + s], O.cw_bias[8 * q + 4 + s]);
        const uint32_t ha = __half_as_ushort(__float2half_rn(a)), hb = __half_as_ushort(__float2half_rn(b));
        B.lo[s] = g == 0 ? ha : (g == 1 ? (ha << 16) : 0u);
        B.hi[s] = g == 0 ? hb : (g == 1 ? (hb << 16) : 0u);
    }
    return B;
}

// One m-tile (2 levels) of loads for this lane's corner: 2 lines x 2 chunks of 16 B, plus the
// lane's trilinear corner weights.
struct GatherTile {
    uint32_t v[2][8];   // row g (level 2t) / row g+8 (level 2t+1): members 8q..8q+7, (f0,f1) each
    float w[2];
};

// 32 bytes read-only from global memory as two LDG.128 (sm_90 has no 256-bit load).  The first load of a quad already
// touches all four sectors of the 128 B line, so the second one finds the line in L1.
__device__ __forceinline__ void ldg256(const void *p, uint32_t (&r)[8]) {
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
                 : "l"(p));
}

// -------------------------------------------------------------------------------------------
// Quad-cooperative index computation (warp-specialised kernel).
// The four lanes of a quad (q = 0..3, the four 32 B pieces of one 128 B line) need the same position -> corner ->
// hash/stride -> trilinear-weight arithmetic for their corner g; computed per lane that is 4x redundant, ~80 instructions
// per level and lane, and the gather warps are issue-limited.  Here the 32 lanes compute 32 DISTINCT (level, corner)
// pairs -- lane L: level 4U + (L >> 3), corner L & 7 -- once per four levels, and each tile's issue fetches the two
// (entry, weight) pairs it needs with shuffles.
// -------------------------------------------------------------------------------------------
struct QuadIdx {
    uint32_t entry;   // offset[level] + index: absolute table line of (level 4U + (lane >> 3), corner lane & 7)
    float w;          // its trilinear weight
};

template <int U>
__device__ __forceinline__ QuadIdx quad_compute(const nsb_field_params &P, float x, float y, float z, int lane) {
    const int l = 4 * U + (lane >> 3);   // dynamic index into the __grid_constant__ level table: LDC, no local copy
    const uint32_t dx = lane & 1, dy = (lane >> 1) & 1, dz = (lane >> 2) & 1;
    const float scale = P.levels.scale[l];
    const uint32_t res = P.levels.res[l], ent = P.levels.entries[l], off = P.levels.offset[l];
    const float px = fmaf(scale, x, 0.5f), py = fmaf(scale, y, 0.5f), pz = fmaf(scale, z, 0.5f);
    const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
    const float fx = px - flx, fy = py - fly, fz = pz - flz;
    const uint32_t cx = (uint32_t)(int)flx + dx, cy = (uint32_t)(int)fly + dy, cz = (uint32_t)(int)flz + dz;
    QuadIdx Q;
    Q.w = ((dx ? fx : 1.0f - fx) * (dy ? fy : 1.0f - fy)) * (dz ? fz : 1.0f - fz);
    const uint32_t ih = (cx ^ (cy * kPrimeY) ^ (cz * kPrimeZ)) & (ent - 1);   // hashed levels: entries = 2^log2T
    uint32_t id = cx + cy * res + cz * res * res;                              // < 2*entries: `% entries` is one subtract
    id = id >= ent ? id - ent : id;
    Q.entry = off + (P.levels.hashed[l] ? ih : id);
    return Q;
}

// loads of tile J (0/1) of the quad: line 0 <- level 4U+2J, line 1 <- level 4U+2J+1, corner g
template <int U, int J>
__device__ __forceinline__ void gather_issue_q(const nsb_field_params &P, const uint8_t *tab, const QuadIdx &Q, int g,
                                               GatherTile &G) {
    const uint32_t e0 = __shfl_sync(0xffffffffu, Q.entry, (2 * J) * 8 + g);
    const uint32_t e1 = __shfl_sync(0xffffffffu, Q.entry, (2 * J + 1) * 8 + g);
    G.w[0] = __shfl_sync(0xffffffffu, Q.w, (2 * J) * 8 + g);
    G.w[1] = __shfl_sync(0xffffffffu, Q.w, (2 * J + 1) * 8 + g);
    ldg256(tab + (size_t)e0 * 128, G.v[0]);
    ldg256(tab + (size_t)e1 * 128, G.v[1]);
}

// Software-pipelined gather of one sample, quad-cooperative.  On entry Ga holds the loads of this sample's tile 0
// and Q its quad 0; on return they hold the NEXT sample's (when next_xs != nullptr; next_out = that sample's smem row).
// The 8 lanes (q == 0) that own a level quad's features store them to the shared-memory feature row as soon as the
// quad is reduced (no yv[4] carried to a final 4-shuffle delivery), and the next sample's position is read from
// shared memory when its first loads are issued (not held across the body): register pressure in the gather role is
// what decides its speed, and a spill inside this loop is very expensive (L1 is flooded by the streaming table lines).
// (Tried and dropped: feeding the HMMA A fragment straight from the load registers -- m16 row halves = even / odd
// members of ONE line -- takes fewer instructions per sample but puts an extra shuffle per level on the per-warp
// dependent chain, and the loop is latency-, not issue-bound.)
// B fragments parked in a lane-private shared-memory column ([k-step][lane] uint2 = {b0, b1}) and fetched one k-step
// at a time: rebuilt only when the timestep changes, and 8 registers that are not live across the sample loop.
struct BlendBSmem {
    const uint2 *col;   // this lane's column: col[s * 32]
};
__device__ __forceinline__ void park_blend_b(const BlendB &B, uint2 *warp_slot, int lane) {
#pragma unroll
    for (int s = 0; s < 4; ++s) warp_slot[s * 32 + lane] = make_uint2(B.lo[s], B.hi[s]);
}
// cv (training forward only): the member-blended value of each corner BEFORE the trilinear weight, fp16 pairs
// [level][corner] -- what the position gradient needs (d w / d x times the blended corner value), saved so that
// the backward does not gather the table lines a second time.  cv points at this tile's two levels.
__device__ __forceinline__ float gather_consume(const GatherTile &G, const BlendBSmem &B, int lane, __half2 *cv = nullptr) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const uint2 b = B.col[s * 32];
        const uint32_t a[4] = {G.v[0][s], G.v[1][s], G.v[0][4 + s], G.v[1][4 + s]};
        mma16816(c, a, b.x, b.y);
    }
    if (cv && (lane & 3) == 0) {
        cv[lane >> 2] = __floats2half2_rn(c[0], c[1]);
        cv[8 + (lane >> 2)] = __floats2half2_rn(c[2], c[3]);
    }
    const float u0 = butterfly(c[0] * G.w[0], c[1] * G.w[0], 2, lane);
    const float u1 = butterfly(c[2] * G.w[1], c[3] * G.w[1], 2, lane);
    return butterfly(u0, u1, 3, lane);
}

template <bool CV, class BT>
__device__ __forceinline__ void gather_sample_quad(const nsb_field_params &P, const uint8_t *tab, float x, float y,
                                                   float z, const float4 *next_xs, float4 &next_out, const BT &B,
                                                   GatherTile &Ga, QuadIdx &Q, __half *feat_row, __half2 *cv_row, int lane) {
    const int g = lane >> 2;
    const bool owner = (lane & 3) == 0;
    GatherTile Gb;
    float e, o, yv;
    gather_issue_q<0, 1>(P, tab, Q, g, Gb); e = gather_consume(Ga, B, lane, CV ? cv_row + 0 : nullptr);
    Q = quad_compute<1>(P, x, y, z, lane);
    gather_issue_q<1, 0>(P, tab, Q, g, Ga); o = gather_consume(Gb, B, lane, CV ? cv_row + 16 : nullptr); yv = butterfly(e, o, 4, lane);
    if (owner) feat_row[g] = __float2half_rn(yv);
    gather_issue_q<1, 1>(P, tab, Q, g, Gb); e = gather_consume(Ga, B, lane, CV ? cv_row + 32 : nullptr);
    Q = quad_compute<2>(P, x, y, z, lane);
    gather_issue_q<2, 0>(P, tab, Q, g, Ga); o = gather_consume(Gb, B, lane, CV ? cv_row + 48 : nullptr); yv = butterfly(e, o, 4, lane);
    if (owner) feat_row[8 + g] = __float2half_rn(yv);
    gather_issue_q<2, 1>(P, tab, Q, g, Gb); e = gather_consume(Ga, B, lane, CV ? cv_row + 64 : nullptr);
    Q = quad_compute<3>(P, x, y, z, lane);
    gather_issue_q<3, 0>(P, tab, Q, g, Ga); o = gather_consume(Gb, B, lane, CV ? cv_row + 80 : nullptr); yv = butterfly(e, o, 4, lane);
    if (owner) feat_row[16 + g] = __float2half_rn(yv);
    gather_issue_q<3, 1>(P, tab, Q, g, Gb); e = gather_consume(Ga, B, lane, CV ? cv_row + 96 : nullptr);
    if (next_xs) {
        next_out = *next_xs;
        Q = quad_compute<0>(P, next_out.x, next_out.y, next_out.z, lane);
        gather_issue_q<0, 0>(P, tab, Q, g, Ga);
    }
    o = gather_consume(Gb, B, lane, CV ? cv_row + 112 : nullptr); yv = butterfly(e, o, 4, lane);
    if (owner) feat_row[24 + g] = __float2half_rn(yv);
}

}  // namespace nsb
