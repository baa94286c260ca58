// Isosurface extraction from a density grid: marching tetrahedra on the Kuhn split (nsb_mesh_count / nsb_mesh_emit).
//
// Pass structure (DESIGN 4.2d): count (per-point crossing masks, per-tile vertex / face sums) | exclusive scan of the tile
// sums | vertices (per-point vertex ids, positions) | faces.  Every output position comes from a block scan over a fixed
// point order plus the scanned tile offset: no atomics, the output is the same bits on every run.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <cmath>

#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kMeshThreads = 256;
constexpr int kMeshItems = NSB_MESH_TILE / kMeshThreads;     // points per thread; item k of thread t: k * 256 + t
constexpr int kScanThreads = 512;
static_assert(NSB_MESH_TILE % kMeshThreads == 0, "tile");

// Cube corners and edge directions as 3-bit masks: bit 0 = +x, bit 1 = +y, bit 2 = +z.
// Slot of an edge direction, in the owner's slot order +x, +y, +z, +x+y, +x+z, +y+z, +x+y+z.
__constant__ int8_t kSlotOfDir[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
__constant__ uint8_t kDirOfSlot[7] = {1, 2, 4, 3, 5, 6, 7};
// Kuhn tetrahedra, one per axis permutation (a, b, c) in the order (x,y,z), (x,z,y), (y,x,z), (y,z,x), (z,x,y), (z,y,x):
// corners 0, e_a, e_a + e_b, 111.  Parity = sign of the permutation = orientation of (v0, v1, v2, v3).
__constant__ uint8_t kTet[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ int8_t kTetParity[6] = {1, -1, -1, 1, 1, -1};

struct Grid {
    int nx, ny, nz;
    int64_t plane;      // nx * ny
};

__device__ __forceinline__ Grid grid_of(const nsb_mesh_args &A) {
    return Grid{(int)A.nx, (int)A.ny, (int)A.nz, A.nx * A.ny};
}

// Bits of the corner directions that exist at point (x, y, z): bit d set iff the point + d is on the grid.
__device__ __forceinline__ uint32_t valid_dirs(const Grid &g, int x, int y, int z) {
    const bool vx = x + 1 < g.nx, vy = y + 1 < g.ny, vz = z + 1 < g.nz;
    uint32_t v = 0;
#pragma unroll
    for (int d = 0; d < 8; ++d)
        if ((!(d & 1) || vx) && (!(d & 2) || vy) && (!(d & 4) || vz)) v |= 1u << d;
    return v;
}

__device__ __forceinline__ int64_t dir_offset(const Grid &g, int d) {
    return (d & 1) + ((d & 2) ? (int64_t)g.nx : 0) + ((d & 4) ? g.plane : 0);
}

// Triangles of a tetrahedron with n of its 4 corners inside.
__device__ __forceinline__ int tri_count(int n) { return (n == 1 || n == 3) ? 1 : (n == 2 ? 2 : 0); }

// Faces of the cell whose lowest corner has inside bits `in8` (bit c: corner c inside).
__device__ __forceinline__ int cell_faces(uint32_t in8) {
    int f = 0;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        int n = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) n += (in8 >> kTet[t][c]) & 1u;
        f += tri_count(n);
    }
    return f;
}

__device__ __forceinline__ void point_coords(const Grid &g, int64_t i, int &x, int &y, int &z) {
    z = (int)(i / g.plane);
    const int64_t r = i - (int64_t)z * g.plane;
    y = (int)(r / g.nx);
    x = (int)(r - (int64_t)y * g.nx);
}

// ---------------------------------------------------------------------------------------------
// count: point_mask[i] = crossing slots (bits 0-6) | inside (bit 7); tile_sums[2b] = vertices, [2b+1] = faces of tile b
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMeshThreads) mesh_count_kernel(const __grid_constant__ nsb_mesh_args A) {
    using Reduce = cub::BlockReduce<int, kMeshThreads>;
    __shared__ typename Reduce::TempStorage tmp_v, tmp_f;
    const Grid g = grid_of(A);
    const int64_t n = g.plane * g.nz;
    const int64_t base = (int64_t)blockIdx.x * NSB_MESH_TILE;
    int nv = 0, nf = 0;
#pragma unroll 1
    for (int k = 0; k < kMeshItems; ++k) {
        const int64_t i = base + k * kMeshThreads + threadIdx.x;
        if (i >= n) break;
        int x, y, z;
        point_coords(g, i, x, y, z);
        const uint32_t valid = valid_dirs(g, x, y, z);
        uint32_t in8 = 0;
#pragma unroll
        for (int d = 0; d < 8; ++d)
            if ((valid >> d) & 1u) in8 |= (A.sigma[i + dir_offset(g, d)] > A.level ? 1u : 0u) << d;
        const uint32_t in0 = in8 & 1u;
        uint32_t mask = in0 << 7;
#pragma unroll
        for (int s = 0; s < 7; ++s) {
            const int d = kDirOfSlot[s];
            if (((valid >> d) & 1u) && ((in8 >> d) & 1u) != in0) mask |= 1u << s;
        }
        A.point_mask[i] = (uint8_t)mask;
        nv += __popc(mask & 0x7fu);
        if (valid == 0xffu) nf += cell_faces(in8);
    }
    const int sv = Reduce(tmp_v).Sum(nv);
    const int sf = Reduce(tmp_f).Sum(nf);
    if (threadIdx.x == 0) {
        A.tile_sums[2 * blockIdx.x] = sv;
        A.tile_sums[2 * blockIdx.x + 1] = sf;
    }
}

// Exclusive scan of the (vertices, faces) tile sums in place, totals after them.  One CTA: each thread sums a contiguous
// run of tiles, a block scan over the run sums, then each thread rewrites its run.
__global__ void __launch_bounds__(kScanThreads) mesh_scan_kernel(int64_t *tile_sums, int64_t n_tiles) {
    using Scan = cub::BlockScan<long long, kScanThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t per = (n_tiles + kScanThreads - 1) / kScanThreads;
    const int64_t lo = min((int64_t)threadIdx.x * per, n_tiles), hi = min(lo + per, n_tiles);
    long long run[2] = {0, 0};
    for (int64_t b = lo; b < hi; ++b) {
        run[0] += tile_sums[2 * b];
        run[1] += tile_sums[2 * b + 1];
    }
    long long ex[2], tot[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        Scan(tmp).ExclusiveSum(run[j], ex[j], tot[j]);
        __syncthreads();
    }
    for (int64_t b = lo; b < hi; ++b) {
        const long long v = tile_sums[2 * b], f = tile_sums[2 * b + 1];
        tile_sums[2 * b] = ex[0];
        tile_sums[2 * b + 1] = ex[1];
        ex[0] += v;
        ex[1] += f;
    }
    if (threadIdx.x == 0) {
        tile_sums[2 * n_tiles] = tot[0];
        tile_sums[2 * n_tiles + 1] = tot[1];
    }
}

// World coordinate of grid index i on one axis: box_min + i * h, rounded after each operation.
__device__ __forceinline__ float grid_coord(float box_min, float h, int i) {
    return __fadd_rn(box_min, __fmul_rn((float)i, h));
}

// ---------------------------------------------------------------------------------------------
// vertices: vertex_base[i] = id of point i's first vertex; one vertex per crossing slot, in slot order
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMeshThreads) mesh_vertices_kernel(const __grid_constant__ nsb_mesh_args A) {
    using Scan = cub::BlockScan<int, kMeshThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const Grid g = grid_of(A);
    const int64_t n = g.plane * g.nz;
    const int64_t base = (int64_t)blockIdx.x * NSB_MESH_TILE;
    int64_t next = A.tile_sums[2 * blockIdx.x];
#pragma unroll 1
    for (int k = 0; k < kMeshItems; ++k) {
        const int64_t i = base + k * kMeshThreads + threadIdx.x;
        const uint32_t mask = i < n ? A.point_mask[i] : 0u;
        int ex, tot;
        Scan(tmp).ExclusiveSum(__popc(mask & 0x7fu), ex, tot);
        __syncthreads();
        if (i < n) {
            const int64_t first = next + ex;
            A.vertex_base[i] = (int32_t)first;
            if (mask & 0x7fu) {
                int x, y, z;
                point_coords(g, i, x, y, z);
                const float s0 = A.sigma[i];
                const float p0[3] = {grid_coord(A.box_min[0], A.h[0], x), grid_coord(A.box_min[1], A.h[1], y),
                                     grid_coord(A.box_min[2], A.h[2], z)};
                int64_t id = first;
#pragma unroll 1
                for (int s = 0; s < 7; ++s) {
                    if (!((mask >> s) & 1u)) continue;
                    const int d = kDirOfSlot[s];
                    const float s1 = A.sigma[i + dir_offset(g, d)];
                    const float t = __fdiv_rn(__fsub_rn(A.level, s0), __fsub_rn(s1, s0));
                    const float p1[3] = {(d & 1) ? grid_coord(A.box_min[0], A.h[0], x + 1) : p0[0],
                                         (d & 2) ? grid_coord(A.box_min[1], A.h[1], y + 1) : p0[1],
                                         (d & 4) ? grid_coord(A.box_min[2], A.h[2], z + 1) : p0[2]};
                    if (id < A.n_vertices) {
#pragma unroll
                        for (int c = 0; c < 3; ++c)
                            A.vertices[3 * id + c] = __fadd_rn(p0[c], __fmul_rn(t, __fsub_rn(p1[c], p0[c])));
                    }
                    ++id;
                }
            }
        }
        next += tot;
    }
}

// ---------------------------------------------------------------------------------------------
// faces of each cell, in (cell, tetrahedron, triangle) order.  Orientation (DESIGN 4.2d): with tetrahedron corners
// 0..3, parity P and the inside corners known, for the sorted corner lists below
//   1 inside  i, others j<k<l:   (ij, ik, il) if (-1)^i P > 0, else (ij, il, ik)
//   3 inside, outside o, j<k<l:  (oj, ok, ol) if (-1)^o P < 0, else (oj, ol, ok)
//   2 inside i<j, outside k<l:   (ik, il, jl), (ik, jl, jk) if (-1)^(i+j+1) P > 0, else (ik, jk, jl), (ik, jl, il)
// ---------------------------------------------------------------------------------------------
struct CellCtx {
    int64_t i;              // the cell's lowest grid point
    uint32_t masks[8];      // point_mask of the 8 corners
};

__device__ __forceinline__ int32_t edge_vertex(const nsb_mesh_args &A, const Grid &g, const CellCtx &c, int ca, int cb) {
    const int lo = ca & cb, d = ca ^ cb;
    const int slot = kSlotOfDir[d];
    const uint32_t m = c.masks[lo];
    return A.vertex_base[c.i + dir_offset(g, lo)] + __popc(m & ((1u << slot) - 1u));
}

__device__ __forceinline__ void put_face(const nsb_mesh_args &A, int64_t f, int32_t a, int32_t b, int32_t c) {
    if (f < A.n_faces) {
        A.faces[3 * f + 0] = a;
        A.faces[3 * f + 1] = b;
        A.faces[3 * f + 2] = c;
    }
}

__global__ void __launch_bounds__(kMeshThreads) mesh_faces_kernel(const __grid_constant__ nsb_mesh_args A) {
    using Scan = cub::BlockScan<int, kMeshThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const Grid g = grid_of(A);
    const int64_t n = g.plane * g.nz;
    const int64_t base = (int64_t)blockIdx.x * NSB_MESH_TILE;
    int64_t next = A.tile_sums[2 * blockIdx.x + 1];
#pragma unroll 1
    for (int k = 0; k < kMeshItems; ++k) {
        CellCtx c;
        c.i = base + k * kMeshThreads + threadIdx.x;
        uint32_t in8 = 0;
        bool cell = false;
        if (c.i < n) {
            int x, y, z;
            point_coords(g, c.i, x, y, z);
            cell = x + 1 < g.nx && y + 1 < g.ny && z + 1 < g.nz;
        }
        if (cell) {
#pragma unroll
            for (int d = 0; d < 8; ++d) {
                c.masks[d] = A.point_mask[c.i + dir_offset(g, d)];
                in8 |= (c.masks[d] >> 7) << d;
            }
        }
        const int nf = cell ? cell_faces(in8) : 0;
        int ex, tot;
        Scan(tmp).ExclusiveSum(nf, ex, tot);
        __syncthreads();
        if (nf > 0) {
            int64_t f = next + ex;
#pragma unroll 1
            for (int t = 0; t < 6; ++t) {
                int cin[4], cout[4], ni = 0, no = 0;     // local corner indices 0..3, ascending
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if ((in8 >> kTet[t][q]) & 1u) cin[ni++] = q;
                    else cout[no++] = q;
                }
                if (ni == 0 || ni == 4) continue;
                const int P = kTetParity[t];
                const uint8_t *v = kTet[t];
                if (ni == 1 || ni == 3) {
                    // the lone corner and the other three, ascending
                    const int lone = ni == 1 ? cin[0] : cout[0];
                    const int *rest = ni == 1 ? cout : cin;
                    const int sgn = ((lone & 1) ? -P : P) * (ni == 1 ? 1 : -1);
                    const int32_t a = edge_vertex(A, g, c, v[lone], v[rest[0]]);
                    const int32_t b = edge_vertex(A, g, c, v[lone], v[rest[1]]);
                    const int32_t e = edge_vertex(A, g, c, v[lone], v[rest[2]]);
                    if (sgn > 0) put_face(A, f, a, b, e);
                    else put_face(A, f, a, e, b);
                    ++f;
                } else {
                    const int i = cin[0], j = cin[1], kk = cout[0], l = cout[1];
                    const int sgn = ((i + j + 1) & 1) ? -P : P;
                    const int32_t ik = edge_vertex(A, g, c, v[i], v[kk]);
                    const int32_t il = edge_vertex(A, g, c, v[i], v[l]);
                    const int32_t jk = edge_vertex(A, g, c, v[j], v[kk]);
                    const int32_t jl = edge_vertex(A, g, c, v[j], v[l]);
                    if (sgn > 0) {
                        put_face(A, f, ik, il, jl);
                        put_face(A, f + 1, ik, jl, jk);
                    } else {
                        put_face(A, f, ik, jk, jl);
                        put_face(A, f + 1, ik, jl, il);
                    }
                    f += 2;
                }
            }
        }
        next += tot;
    }
}

int64_t mesh_tiles(const nsb_mesh_args *a) { return (a->nx * a->ny * a->nz + NSB_MESH_TILE - 1) / NSB_MESH_TILE; }

int check_mesh_args(const char *who, const nsb_mesh_args *a) {
    if (!a) { set_error("%s: null argument", who); return 1; }
    if (a->nx < 2 || a->ny < 2 || a->nz < 2) { set_error("%s: every grid dimension must be >= 2", who); return 1; }
    if (a->nx >= (1ll << 31) || a->ny >= (1ll << 31) || a->nz >= (1ll << 31) ||
        (double)a->nx * (double)a->ny * (double)a->nz >= 2147483648.0) {
        set_error("%s: the grid must have fewer than 2^31 points", who);
        return 1;
    }
    if (!std::isfinite(a->level)) { set_error("%s: level must be finite", who); return 1; }
    if (!a->sigma || !a->point_mask || !a->tile_sums) { set_error("%s: sigma, point_mask and tile_sums are required", who); return 1; }
    return 0;
}

}  // namespace
}  // namespace nsb

using namespace nsb;

extern "C" int nsb_mesh_count(const nsb_mesh_args *args, void *stream) {
    if (check_mesh_args("nsb_mesh_count", args)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t tiles = mesh_tiles(args);
    mesh_count_kernel<<<(unsigned)tiles, kMeshThreads, 0, st>>>(*args);
    int rc = check_launch("mesh_count_kernel");
    if (rc) return rc;
    mesh_scan_kernel<<<1, kScanThreads, 0, st>>>(args->tile_sums, tiles);
    return check_launch("mesh_scan_kernel");
}

extern "C" int nsb_mesh_emit(const nsb_mesh_args *args, void *stream) {
    if (check_mesh_args("nsb_mesh_emit", args)) return 1;
    if (args->n_vertices < 0 || args->n_faces < 0 || args->n_vertices >= (1ll << 31) || args->n_faces >= (1ll << 31)) {
        set_error("nsb_mesh_emit: n_vertices and n_faces must be in [0, 2^31)");
        return 1;
    }
    if (!args->vertex_base || (args->n_vertices > 0 && !args->vertices) || (args->n_faces > 0 && !args->faces)) {
        set_error("nsb_mesh_emit: vertex_base, vertices and faces are required");
        return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned tiles = (unsigned)mesh_tiles(args);
    mesh_vertices_kernel<<<tiles, kMeshThreads, 0, st>>>(*args);
    int rc = check_launch("mesh_vertices_kernel");
    if (rc || args->n_faces == 0) return rc;
    mesh_faces_kernel<<<tiles, kMeshThreads, 0, st>>>(*args);
    return check_launch("mesh_faces_kernel");
}
