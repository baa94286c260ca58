// Scene flow and optical flow of a render between timesteps (nsb_flow_select / nsb_flow_composite; DESIGN 4.2f).
//
// select:    per-ray counts of the packed samples with weight >= min_weight | exclusive scan of the per-tile sums |
//            fill (sample index, canonical target c = x + offset, init x) in (ray, sample) order.  Every output position
//            is the scanned tile offset, plus a block scan over the tile's rays, plus the sample's rank within its ray
//            (a ballot popcount): no atomics, the same bits on every run.  The selected count is written on the device, ready for nsb_samples.n_samples_dev.
// composite: per ray, the weighted mean of x' - x (and of the projected motion) over its converged selected samples,
//            summed in selection order in fp32.
// Both passes give each ray one warp, so that the lanes read consecutive samples.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <cmath>

#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kFlowThreads = 256;
constexpr int kFlowWarps = kFlowThreads / 32;
constexpr int kScanThreads = 512;
constexpr unsigned kFull = 0xffffffffu;
static_assert(NSB_FLOW_TILE <= kFlowThreads && NSB_FLOW_TILE % kFlowWarps == 0, "tile");

// Packed samples the render produced: slots at or past it are garbage.
__device__ __forceinline__ int64_t flow_n_total(const nsb_flow_select_args &A) {
    return min(*A.n_total, A.capacity);
}

// The packed-sample range [start, end) of ray r, clipped to the render's sample count.
__device__ __forceinline__ void flow_segment(const nsb_flow_select_args &A, int64_t r, int64_t n_total, int64_t &start,
                                             int64_t &end) {
    start = A.packed_info[2 * r];
    end = min(start + A.packed_info[2 * r + 1], n_total);
}

// One warp per ray: each 32-sample chunk of the segment is read by consecutive lanes, and the selection mask of the
// chunk is a ballot, so a sample's rank within its ray is the popcount of the lower lanes' bits: ordered, no atomics.
__device__ __forceinline__ unsigned flow_ballot(const nsb_flow_select_args &A, int64_t i, int64_t end) {
    return __ballot_sync(kFull, i < end && A.weights[i] >= A.min_weight);
}

// ---------------------------------------------------------------------------------------------
// count: ray_sel[r].count = selected samples of ray r; tile_sums[b] = selected samples of tile b
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kFlowThreads) flow_count_kernel(const __grid_constant__ nsb_flow_select_args A) {
    using Reduce = cub::BlockReduce<long long, kFlowThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    const int64_t n_total = flow_n_total(A);
    const int64_t base = (int64_t)blockIdx.x * NSB_FLOW_TILE;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    long long sum = 0;
#pragma unroll 1
    for (int q = warp; q < NSB_FLOW_TILE; q += kFlowWarps) {
        const int64_t r = base + q;
        if (r >= A.n_rays) break;
        int64_t start, end;
        flow_segment(A, r, n_total, start, end);
        int64_t c = 0;
        for (int64_t i0 = start; i0 < end; i0 += 32) c += __popc(flow_ballot(A, i0 + lane, end));
        if (lane == 0) A.ray_sel[2 * r + 1] = c;
        sum += c;
    }
    const long long s = Reduce(tmp).Sum(lane == 0 ? sum : 0);
    if (threadIdx.x == 0) A.tile_sums[blockIdx.x] = s;
}

// Exclusive scan of the tile sums in place, the total into *n_selected.  One CTA: each thread sums a contiguous run of
// tiles, a block scan over the run sums, then each thread rewrites its run.
__global__ void __launch_bounds__(kScanThreads) flow_scan_kernel(int64_t *tile_sums, int64_t n_tiles, int64_t *n_selected) {
    using Scan = cub::BlockScan<long long, kScanThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t per = (n_tiles + kScanThreads - 1) / kScanThreads;
    const int64_t lo = min((int64_t)threadIdx.x * per, n_tiles), hi = min(lo + per, n_tiles);
    long long run = 0;
    for (int64_t b = lo; b < hi; ++b) run += tile_sums[b];
    long long ex, tot;
    Scan(tmp).ExclusiveSum(run, ex, tot);
    for (int64_t b = lo; b < hi; ++b) {
        const long long v = tile_sums[b];
        tile_sums[b] = ex;
        ex += v;
    }
    if (threadIdx.x == 0) *n_selected = tot;
}

// ---------------------------------------------------------------------------------------------
// fill: ray_sel[r].start from a block scan of the tile's counts, then one warp per ray writes its selected samples
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kFlowThreads) flow_fill_kernel(const __grid_constant__ nsb_flow_select_args A) {
    using Scan = cub::BlockScan<long long, kFlowThreads>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ long long first[NSB_FLOW_TILE];
    const int64_t n_total = flow_n_total(A);
    const int64_t base = (int64_t)blockIdx.x * NSB_FLOW_TILE;
    {
        const int64_t r = base + threadIdx.x;
        const bool mine = threadIdx.x < NSB_FLOW_TILE && r < A.n_rays;
        long long ex;
        Scan(tmp).ExclusiveSum(mine ? A.ray_sel[2 * r + 1] : 0, ex);
        ex += A.tile_sums[blockIdx.x];
        if (threadIdx.x < NSB_FLOW_TILE) first[threadIdx.x] = ex;
        if (mine) A.ray_sel[2 * r] = ex;
    }
    __syncthreads();
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const unsigned below = (1u << lane) - 1u;
#pragma unroll 1
    for (int q = warp; q < NSB_FLOW_TILE; q += kFlowWarps) {
        const int64_t r = base + q;
        if (r >= A.n_rays) break;
        int64_t start, end;
        flow_segment(A, r, n_total, start, end);
        int64_t j0 = first[q];
        const float o[3] = {A.origins[3 * r], A.origins[3 * r + 1], A.origins[3 * r + 2]};
        const float d[3] = {A.directions[3 * r], A.directions[3 * r + 1], A.directions[3 * r + 2]};
        for (int64_t i0 = start; i0 < end; i0 += 32) {
            const int64_t i = i0 + lane;
            const unsigned m = flow_ballot(A, i, end);
            if ((m >> lane) & 1u) {
                const int64_t j = j0 + __popc(m & below);
                const float mid = __fadd_rn(A.t_starts[i], A.t_ends[i]);
                A.sel_index[j] = i;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const float x = ray_midpoint(o[a], d[a], mid);
                    A.init[3 * j + a] = x;
                    A.targets[3 * j + a] = __fadd_rn(x, A.offsets[3 * i + a]);
                }
            }
            j0 += __popc(m);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// composite: one warp per ray.  Lanes evaluate consecutive selected samples; every lane then adds the chunk's
// contributions in selection order (broadcast by shuffles), so the sums are sequential and the same bits on every run.
// ---------------------------------------------------------------------------------------------
struct FlowCamera {
    float fx, fy;
    float rot[9];       // camera_to_world rotation, row-major
    float origin[3];
};

// Xc = R^T v (R the camera-to-world rotation).
__device__ __forceinline__ void flow_to_camera(const FlowCamera &cam, const float v[3], float xc[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) xc[k] = cam.rot[k] * v[0] + cam.rot[3 + k] * v[1] + cam.rot[6 + k] * v[2];
}

__global__ void __launch_bounds__(kFlowThreads) flow_composite_kernel(const __grid_constant__ nsb_flow_composite_args A,
                                                                       const FlowCamera cam) {
    const int lane = threadIdx.x % 32;
    const int64_t r = ((int64_t)blockIdx.x * kFlowThreads + threadIdx.x) / 32;
    if (r >= A.n_rays) return;
    const int64_t start = A.ray_sel[2 * r], end = start + A.ray_sel[2 * r + 1];
    const bool camera = A.optical_flow != nullptr;
    float W = 0.f, s[3] = {0.f, 0.f, 0.f};
    float Wp = 0.f, f[2] = {0.f, 0.f};
    for (int64_t j0 = start; j0 < end; j0 += 32) {
        const int64_t j = j0 + lane;
        // this lane's sample: its weight w (0 unless converged), w (x' - x), and for the camera w_p and w_p (pi(x') - pi(x))
        float w = 0.f, c[3] = {0.f, 0.f, 0.f}, wp = 0.f, g[2] = {0.f, 0.f};
        if (j < end && A.status[j] == NSB_INV_CONVERGED) {
            w = A.weights[A.sel_index[j]];
            const float x[3] = {A.init[3 * j], A.init[3 * j + 1], A.init[3 * j + 2]};
            const float dx[3] = {A.positions[3 * j] - x[0], A.positions[3 * j + 1] - x[1], A.positions[3 * j + 2] - x[2]};
#pragma unroll
            for (int k = 0; k < 3; ++k) c[k] = w * dx[k];
            if (camera) {
                // pi(x') - pi(x) from the camera-space motion e = R^T (x' - x), without subtracting two projections:
                // with a = Xc.x, b = Xc.y, z = -Xc.z of x and z' = z - e.z of x',
                //   u' - u = (z e.x + a e.z) / (z z'),  v' - v = (z e.y + b e.z) / (z z')
                const float p[3] = {x[0] - cam.origin[0], x[1] - cam.origin[1], x[2] - cam.origin[2]};
                float xc[3], e[3];
                flow_to_camera(cam, p, xc);
                flow_to_camera(cam, dx, e);
                const float z = -xc[2], z1 = z - e[2];
                if (z > 0.f && z1 > 0.f) {
                    const float q = 1.f / (z * z1);
                    wp = w;
                    g[0] = w * (cam.fx * ((z * e[0] + xc[0] * e[2]) * q));
                    g[1] = w * (-cam.fy * ((z * e[1] + xc[1] * e[2]) * q));
                }
            }
        }
        const int n = (int)min(end - j0, (int64_t)32);
        for (int l = 0; l < n; ++l) {
            W += __shfl_sync(kFull, w, l);
#pragma unroll
            for (int k = 0; k < 3; ++k) s[k] += __shfl_sync(kFull, c[k], l);
            if (camera) {
                Wp += __shfl_sync(kFull, wp, l);
                f[0] += __shfl_sync(kFull, g[0], l);
                f[1] += __shfl_sync(kFull, g[1], l);
            }
        }
    }
    if (lane != 0) return;
    const float iw = W > 0.f ? 1.f / W : 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) A.scene_flow[3 * r + k] = s[k] * iw;
    A.flow_weight[r] = W;
    if (camera) {
        const float ip = Wp > 0.f ? 1.f / Wp : 0.f;
        A.optical_flow[2 * r] = f[0] * ip;
        A.optical_flow[2 * r + 1] = f[1] * ip;
    }
}

int64_t flow_tiles(int64_t n_rays) { return (n_rays + NSB_FLOW_TILE - 1) / NSB_FLOW_TILE; }

}  // namespace
}  // namespace nsb

using namespace nsb;

extern "C" int nsb_flow_select(const nsb_flow_select_args *args, void *stream) {
    const char *who = "nsb_flow_select";
    if (!args) { set_error("%s: null argument", who); return 1; }
    if (args->n_rays < 0) { set_error("%s: n_rays must be >= 0", who); return 1; }
    if (args->capacity <= 0) { set_error("%s: capacity must be > 0", who); return 1; }
    if (!std::isfinite(args->min_weight) || args->min_weight < 0.f || args->min_weight >= 1.f) {
        set_error("%s: min_weight must be finite and in [0, 1)", who);
        return 1;
    }
    if (!args->packed_info || !args->t_starts || !args->t_ends || !args->weights || !args->offsets || !args->origins ||
        !args->directions || !args->n_total || !args->ray_sel || !args->sel_index || !args->targets || !args->init ||
        !args->n_selected || !args->tile_sums) {
        set_error("%s: null pointer", who);
        return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t tiles = flow_tiles(args->n_rays);
    if (tiles > 0) {
        flow_count_kernel<<<(unsigned)tiles, kFlowThreads, 0, st>>>(*args);
        int rc = check_launch("flow_count_kernel");
        if (rc) return rc;
    }
    flow_scan_kernel<<<1, kScanThreads, 0, st>>>(args->tile_sums, tiles, args->n_selected);
    int rc = check_launch("flow_scan_kernel");
    if (rc || tiles == 0) return rc;
    flow_fill_kernel<<<(unsigned)tiles, kFlowThreads, 0, st>>>(*args);
    return check_launch("flow_fill_kernel");
}

extern "C" int nsb_flow_composite(const nsb_flow_composite_args *args, void *stream) {
    const char *who = "nsb_flow_composite";
    if (!args) { set_error("%s: null argument", who); return 1; }
    if (args->n_rays < 0) { set_error("%s: n_rays must be >= 0", who); return 1; }
    if (args->capacity <= 0) { set_error("%s: capacity must be > 0", who); return 1; }
    if (!args->ray_sel || !args->sel_index || !args->init || !args->positions || !args->status || !args->weights ||
        !args->scene_flow || !args->flow_weight) {
        set_error("%s: null pointer", who);
        return 1;
    }
    FlowCamera cam = {};
    if (args->optical_flow) {
        for (int k = 0; k < 4; ++k)
            if (!std::isfinite(args->intrinsics[k])) { set_error("%s: camera values must be finite", who); return 1; }
        for (int k = 0; k < 12; ++k)
            if (!std::isfinite(args->camera_to_world[k])) { set_error("%s: camera values must be finite", who); return 1; }
        if (!(args->intrinsics[0] > 0.f) || !(args->intrinsics[1] > 0.f)) {
            set_error("%s: fx and fy must be > 0", who);
            return 1;
        }
        cam.fx = args->intrinsics[0];
        cam.fy = args->intrinsics[1];
        for (int m = 0; m < 3; ++m) {
            for (int k = 0; k < 3; ++k) cam.rot[3 * m + k] = args->camera_to_world[4 * m + k];
            cam.origin[m] = args->camera_to_world[4 * m + 3];
        }
    }
    if (args->n_rays == 0) return 0;
    const unsigned blocks = (unsigned)((args->n_rays + kFlowWarps - 1) / kFlowWarps);
    flow_composite_kernel<<<blocks, kFlowThreads, 0, (cudaStream_t)stream>>>(*args, cam);
    return check_launch("flow_composite_kernel");
}
