// pm_mesh.cu -- TSDF integration of depth maps and marching cubes over a sparse grid of 8^3-voxel blocks (beyond the
// reference; definition in include/patchmatch_b200.h, INTEGRATION.md "Meshes (beyond the reference)", DESIGN.md K-M).
//
//   allocation   per seed point the keys of the (up to 8) blocks its truncation cube meets -> CUB radix sort -> unique;
//   integration  one CTA of 512 threads per block, one thread per voxel, every view in one launch: the view table is staged
//                in shared memory 32 views at a time, and warp 0 culls each view for the whole block (block behind the
//                camera, or its projection off the image) before the voxels run through the survivors in view order;
//   extraction   each CTA resolves its 26 neighbour blocks (binary search over the sorted keys) and loads a 10^3 tile of
//                its voxels plus a one-voxel halo; a count pass writes per voxel its owned vertices and in-block vertex
//                prefix and per block the totals, CUB scans the block totals, and the write pass emits vertices and faces,
//                reading vertex indices across block borders from the neighbour's prefixes.  An edge owns a vertex only
//                when one of its four cubes is meshed, so no vertex is unreferenced.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_mesh_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmmesh;

constexpr int kBlock = 256;
constexpr int kVoxThreads = kBlockVoxels;         // one thread per voxel of a block
constexpr int kViewChunk = 32;                    // views staged per round (warp 0 culls one per lane)
constexpr long long kMaxPoints = 1ll << 28;       // 8 keys per point stay below 2^31
constexpr long long kMaxBlocks = 1ll << 22;       // voxel indices block * 512 + v stay below 2^31
constexpr int kTile = 10;                         // voxels -1..8 of a block per axis
constexpr int kCubes = 9;                         // cubes with minimum corner -1..7 per axis

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct Carver {  // bump allocator over the caller's workspace; a NULL base only measures
    char *base;
    size_t used = 0;
    template <typename T>
    T *take(size_t count) {
        T *p = base ? reinterpret_cast<T *>(base + used) : nullptr;
        used += align256(count * sizeof(T));
        return p;
    }
};

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 ? 65535 : b));
}

// ---- allocation ------------------------------------------------------------------------------------------------------------

struct AllocLayout {
    unsigned long long *unique;   // at the workspace's start: the result
    unsigned long long *keys_in, *keys_sorted;
    long long *n_unique;
    int *bad;
    void *cub;
    size_t cub_bytes;
};

bool alloc_layout(Carver &c, long long n, AllocLayout &l) {
    const long long m = 8 * (n < 1 ? 1 : n);
    l.unique = c.take<unsigned long long>(m);
    l.keys_in = c.take<unsigned long long>(m);
    l.keys_sorted = c.take<unsigned long long>(m);
    l.n_unique = c.take<long long>(2);
    l.bad = reinterpret_cast<int *>(l.n_unique + 1);
    size_t a = 0, b = 0;
    if (cub::DeviceRadixSort::SortKeys(nullptr, a, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int)m, 0, 63) != cudaSuccess)
        return false;
    if (cub::DeviceSelect::Unique(nullptr, b, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (long long *)nullptr, (int)m) !=
        cudaSuccess)
        return false;
    l.cub_bytes = a > b ? a : b;
    l.cub = c.take<char>(l.cub_bytes);
    return true;
}

// 8 keys per point: every (lo|hi) combination of the block ranges (a block range spans at most 2 blocks since trunc <= 4);
// repeats are removed by the unique pass
__global__ void __launch_bounds__(kBlock) alloc_keys_kernel(const float *p, int n, double s, double tau, unsigned long long *keys,
                                                            int *bad) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        int lo[3], hi[3];
        bool ok = true;
        for (int a = 0; a < 3; ++a) ok = seed_range(p[3 * (size_t)i + a], s, tau, lo[a], hi[a]) && ok;
        if (!ok) {
            *bad = 1;
            for (int c = 0; c < 8; ++c) keys[8 * (size_t)i + c] = 0;
            continue;
        }
        for (int c = 0; c < 8; ++c) {
            const int bi = ((c & 1) ? hi[0] : lo[0]) >> 3, bj = ((c & 2) ? hi[1] : lo[1]) >> 3, bk = ((c & 4) ? hi[2] : lo[2]) >> 3;
            keys[8 * (size_t)i + c] = block_key(bi, bj, bk);
        }
    }
}

// ---- integration -----------------------------------------------------------------------------------------------------------

// false when no voxel centre of the block can land on a pixel of the view: every centre lies in the box lo..hi, so its
// projection lies in the hull of the box corners' projections when they are all in front of the camera
__device__ bool block_may_see(const pmb200_tsdf_view &v, const double *lo, const double *hi) {
    double umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
    int front = 0;
    for (int c = 0; c < 8; ++c) {
        const double x = (c & 1) ? hi[0] : lo[0], y = (c & 2) ? hi[1] : lo[1], z = (c & 4) ? hi[2] : lo[2];
        const double xc = rigid_row(v.Rt, x, y, z), yc = rigid_row(v.Rt + 4, x, y, z), zc = rigid_row(v.Rt + 8, x, y, z);
        if (!(zc > 0.0)) continue;
        ++front;
        const double u = div64(add64(add64(mul64(v.K[0], xc), mul64(v.K[1], yc)), mul64(v.K[2], zc)), zc);
        const double w = div64(add64(add64(mul64(v.K[3], xc), mul64(v.K[4], yc)), mul64(v.K[5], zc)), zc);
        umin = fmin(umin, u); umax = fmax(umax, u); vmin = fmin(vmin, w); vmax = fmax(vmax, w);
    }
    if (front == 0) return false;
    if (front < 8) return true;  // the block straddles the camera plane: keep it
    // a pixel needs -0.5 <= u < W - 0.5; one more pixel of margin absorbs the rounding of the corner projections
    return !(umax < -1.5 || umin > (double)v.width + 0.5 || vmax < -1.5 || vmin > (double)v.height + 0.5);
}

struct IntegrateParams {
    const unsigned long long *keys;
    const pmb200_tsdf_view *views;
    int n_views;
    double s, tau;
    const float *depth, *image;
    float *tsdf, *weight;
    uchar4 *colour;
};

__global__ void __launch_bounds__(kVoxThreads) integrate_kernel(const IntegrateParams p) {
    __shared__ pmb200_tsdf_view sv[kViewChunk];
    __shared__ int live[kViewChunk];
    __shared__ int n_live;
    const int t = threadIdx.x;
    int bi, bj, bk;
    key_block(p.keys[blockIdx.x], bi, bj, bk);
    const double X = voxel_centre(8 * bi + (t & 7), p.s), Y = voxel_centre(8 * bj + ((t >> 3) & 7), p.s),
                 Z = voxel_centre(8 * bk + (t >> 6), p.s);
    const double lo[3] = {voxel_centre(8 * bi, p.s), voxel_centre(8 * bj, p.s), voxel_centre(8 * bk, p.s)};
    const double hi[3] = {voxel_centre(8 * bi + 7, p.s), voxel_centre(8 * bj + 7, p.s), voxel_centre(8 * bk + 7, p.s)};
    VoxelSums acc;
    sums_init(acc);
    for (int c0 = 0; c0 < p.n_views; c0 += kViewChunk) {
        const int cn = p.n_views - c0 < kViewChunk ? p.n_views - c0 : kViewChunk;
        __syncthreads();  // the previous chunk is done with sv / live
        {
            const unsigned long long *src = reinterpret_cast<const unsigned long long *>(p.views + c0);
            unsigned long long *dst = reinterpret_cast<unsigned long long *>(sv);
            const int words = cn * (int)(sizeof(pmb200_tsdf_view) / 8);
            for (int w = t; w < words; w += kVoxThreads) dst[w] = __ldg(src + w);
        }
        __syncthreads();
        if (t < 32) {
            const bool keep = t < cn && block_may_see(sv[t], lo, hi);
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (keep) live[__popc(m & ((1u << t) - 1u))] = t;
            if (t == 0) n_live = __popc(m);
        }
        __syncthreads();
        for (int q = 0; q < n_live; ++q) {
            const pmb200_tsdf_view &v = sv[live[q]];
            const double xc = rigid_row(v.Rt, X, Y, Z), yc = rigid_row(v.Rt + 4, X, Y, Z), zc = rigid_row(v.Rt + 8, X, Y, Z);
            int px, py;
            if (!view_pixel(v.K, v.height, v.width, xc, yc, zc, px, py)) continue;
            const size_t plane = (size_t)v.height * v.width, pix = (size_t)py * v.width + px;
            const float d = __ldg(p.depth + v.depth_offset + pix);
            const float *img = p.image + v.image_offset + pix;
            if (!(d > 0.0f) || !(d < INFINITY) || sub64((double)d, zc) < -p.tau) continue;
            voxel_update(acc, d, zc, p.tau, __ldg(img), __ldg(img + plane), __ldg(img + 2 * plane));
        }
    }
    float ts, w;
    unsigned char rgb[3];
    voxel_finish(acc, ts, w, rgb);
    const size_t g = (size_t)blockIdx.x * kBlockVoxels + t;
    p.tsdf[g] = ts;
    p.weight[g] = w;
    p.colour[g] = make_uchar4(rgb[0], rgb[1], rgb[2], 0);
}

// ---- extraction ------------------------------------------------------------------------------------------------------------

struct MeshLayout {
    unsigned char *info;           // per voxel: owned-edge mask (bits 0..2) | triangles of its cube << 3
    unsigned short *vpre;          // per voxel: owned vertices of the voxels before it in its block
    int *bcount;                   // per block: vertices, then per block: faces ([2][n_blocks])
    long long *vbase, *tbase;      // [n_blocks + 1]: exclusive prefix of the block totals
    void *cub;
    size_t cub_bytes;
};

bool mesh_layout(Carver &c, long long nb, MeshLayout &l) {
    const long long n = nb < 1 ? 1 : nb;
    l.info = c.take<unsigned char>(n * kBlockVoxels);
    l.vpre = c.take<unsigned short>(n * kBlockVoxels);
    l.bcount = c.take<int>(2 * n);
    l.vbase = c.take<long long>(n + 1);
    l.tbase = c.take<long long>(n + 1);
    size_t b = 0;
    if (cub::DeviceScan::InclusiveSum(nullptr, b, (int *)nullptr, (long long *)nullptr, (int)n) != cudaSuccess) return false;
    l.cub_bytes = b;
    l.cub = c.take<char>(b);
    return true;
}

struct MeshParams {
    const unsigned long long *keys;
    int n_blocks;
    const float *tsdf, *weight;
    const uchar4 *colour;
    float min_weight;
    double s;
    MeshLayout l;
    unsigned char *verts;
    int *faces;
};

struct MeshShared {
    int nb[27];                          // neighbour block index or -1, (dx + 1) + 3 (dy + 1) + 9 (dz + 1)
    float tile[kTile * kTile * kTile];   // tsdf of voxels -1..8, NaN when not valid
    short cube[kCubes * kCubes * kCubes];  // cube index of the cubes with minimum corner -1..7, -1 unless all corners valid
    signed char table[256 * kTableWidth];
};

__device__ inline int tile_at(int x, int y, int z) { return (x + 1) + kTile * (y + 1) + kTile * kTile * (z + 1); }
__device__ inline int cube_at(int x, int y, int z) { return (x + 1) + kCubes * (y + 1) + kCubes * kCubes * (z + 1); }
__device__ inline int nb_at(int x, int y, int z) { return ((x >> 3) + 1) + 3 * ((y >> 3) + 1) + 9 * ((z >> 3) + 1); }

// block index of key, or -1
__device__ int find_block(const unsigned long long *keys, int n, unsigned long long key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo < n && __ldg(keys + lo) == key ? lo : -1;
}

__device__ void load_tile(const MeshParams &p, MeshShared &sh) {
    const int t = threadIdx.x;
    if (t < 27) {
        int bi, bj, bk;
        key_block(p.keys[blockIdx.x], bi, bj, bk);
        const long long x = bi + t % 3 - 1, y = bj + (t / 3) % 3 - 1, z = bk + t / 9 - 1;
        const bool inside = x >= -kKeyBias && x < kKeyBias && y >= -kKeyBias && y < kKeyBias && z >= -kKeyBias && z < kKeyBias;
        sh.nb[t] = inside ? find_block(p.keys, p.n_blocks, block_key(x, y, z)) : -1;
    }
    for (int i = t; i < 256 * kTableWidth; i += kVoxThreads) sh.table[i] = kTriTable[i / kTableWidth][i % kTableWidth];
    __syncthreads();
    for (int i = t; i < kTile * kTile * kTile; i += kVoxThreads) {
        const int x = i % kTile - 1, y = (i / kTile) % kTile - 1, z = i / (kTile * kTile) - 1;
        const int b = sh.nb[nb_at(x, y, z)];
        float v = __int_as_float(0x7fc00000);
        if (b >= 0) {
            const size_t g = (size_t)b * kBlockVoxels + (x & 7) + 8 * (y & 7) + 64 * (z & 7);
            if (__ldg(p.weight + g) >= p.min_weight) v = __ldg(p.tsdf + g);
        }
        sh.tile[i] = v;
    }
    __syncthreads();
    for (int i = t; i < kCubes * kCubes * kCubes; i += kVoxThreads) {
        const int x = i % kCubes - 1, y = (i / kCubes) % kCubes - 1, z = i / (kCubes * kCubes) - 1;
        float c[8];
        bool ok = true;
        for (int k = 0; k < 8; ++k) {
            const int o = corner_offset(k);
            c[k] = sh.tile[tile_at(x + (o & 1), y + ((o >> 1) & 1), z + (o >> 2))];
            ok = ok && !isnan(c[k]);
        }
        sh.cube[i] = ok ? (short)cube_index(c) : (short)-1;
    }
    __syncthreads();
}

__device__ inline int triangles_of(const MeshShared &sh, int idx) {
    if (idx <= 0 || idx >= 255) return 0;
    int n = 0;
    while (n < kMaxTriangles && sh.table[idx * kTableWidth + 3 * n] >= 0) ++n;
    return n;
}

// owned-edge mask of voxel (x, y, z) in 0..7: bit k when the edge to the next voxel along axis k changes sign between two
// valid voxels and one of its four cubes is meshed
__device__ int owned_edges(const MeshShared &sh, int x, int y, int z) {
    const float ta = sh.tile[tile_at(x, y, z)];
    int mask = 0;
    if (isnan(ta)) return 0;
    for (int k = 0; k < 3; ++k) {
        const int ex = k == 0, ey = k == 1, ez = k == 2;
        const float tb = sh.tile[tile_at(x + ex, y + ey, z + ez)];
        if (isnan(tb) || (ta < 0.0f) == (tb < 0.0f)) continue;
        // the four cubes: minimum corners a minus 0 or 1 along each of the two other axes
        const int ux = k == 0 ? 0 : 1, uy = k == 1 ? 0 : 1, uz = k == 2 ? 0 : 1;  // axes the cubes step back along
        bool meshed = false;
        for (int q = 0; q < 4; ++q) {
            int dx = 0, dy = 0, dz = 0, bit = 0;
            if (ux) dx = (q >> bit++) & 1;
            if (uy) dy = (q >> bit++) & 1;
            if (uz) dz = (q >> bit++) & 1;
            meshed = meshed || sh.cube[cube_at(x - dx, y - dy, z - dz)] >= 0;
        }
        if (meshed) mask |= 1 << k;
    }
    return mask;
}

__global__ void __launch_bounds__(kVoxThreads) mesh_count_kernel(const MeshParams p) {
    __shared__ MeshShared sh;
    using Scan = cub::BlockScan<int, kVoxThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    load_tile(p, sh);
    const int t = threadIdx.x, x = t & 7, y = (t >> 3) & 7, z = t >> 6;
    const int mask = owned_edges(sh, x, y, z);
    const int ntri = triangles_of(sh, sh.cube[cube_at(x, y, z)]);
    int pre, total;
    Scan(scan_tmp).ExclusiveSum(__popc(mask), pre, total);
    const size_t g = (size_t)blockIdx.x * kBlockVoxels + t;
    p.l.info[g] = (unsigned char)(mask | (ntri << 3));
    p.l.vpre[g] = (unsigned short)pre;
    __syncthreads();
    int tpre, ttotal;
    Scan(scan_tmp).ExclusiveSum(ntri, tpre, ttotal);
    if (t == 0) {
        p.l.bcount[blockIdx.x] = total;
        p.l.bcount[p.n_blocks + blockIdx.x] = ttotal;
    }
}

__device__ inline void put_f32(unsigned char *dst, float v) {
    const unsigned u = __float_as_uint(v);
    dst[0] = u & 0xff; dst[1] = (u >> 8) & 0xff; dst[2] = (u >> 16) & 0xff; dst[3] = u >> 24;
}

__global__ void __launch_bounds__(kVoxThreads) mesh_write_kernel(const MeshParams p) {
    __shared__ MeshShared sh;
    using Scan = cub::BlockScan<int, kVoxThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    load_tile(p, sh);
    const int t = threadIdx.x, x = t & 7, y = (t >> 3) & 7, z = t >> 6;
    const size_t g = (size_t)blockIdx.x * kBlockVoxels + t;
    const int info = p.l.info[g];
    int bi, bj, bk;
    key_block(p.keys[blockIdx.x], bi, bj, bk);
    // vertices of the owned edges
    long long vi = p.l.vbase[blockIdx.x] + p.l.vpre[g];
    if (info & 7) {
        const int ia[3] = {8 * bi + x, 8 * bj + y, 8 * bk + z};
        const double xa[3] = {voxel_centre(ia[0], p.s), voxel_centre(ia[1], p.s), voxel_centre(ia[2], p.s)};
        const float ta = sh.tile[tile_at(x, y, z)];
        const uchar4 ca4 = p.colour[g];
        const unsigned char ca[3] = {ca4.x, ca4.y, ca4.z};
        for (int k = 0; k < 3; ++k) {
            if (!((info >> k) & 1)) continue;
            const int ex = k == 0, ey = k == 1, ez = k == 2;
            const int xb = x + ex, yb = y + ey, zb = z + ez;
            const size_t gb = (size_t)sh.nb[nb_at(xb, yb, zb)] * kBlockVoxels + (xb & 7) + 8 * (yb & 7) + 64 * (zb & 7);
            const double xbw[3] = {voxel_centre(ia[0] + ex, p.s), voxel_centre(ia[1] + ey, p.s), voxel_centre(ia[2] + ez, p.s)};
            const uchar4 cb4 = p.colour[gb];
            const unsigned char cb[3] = {cb4.x, cb4.y, cb4.z};
            float pos[3];
            unsigned char rgb[3];
            edge_vertex(xa, xbw, ta, sh.tile[tile_at(xb, yb, zb)], ca, cb, pos, rgb);
            unsigned char *rec = p.verts + 15 * (size_t)vi;
            put_f32(rec, pos[0]); put_f32(rec + 4, pos[1]); put_f32(rec + 8, pos[2]);
            rec[12] = rgb[0]; rec[13] = rgb[1]; rec[14] = rgb[2];
            ++vi;
        }
    }
    // faces of the cube at this voxel
    const int ntri = info >> 3;
    int tpre, ttotal;
    Scan(scan_tmp).ExclusiveSum(ntri, tpre, ttotal);
    if (ntri == 0) return;
    const int idx = sh.cube[cube_at(x, y, z)];
    int *out = p.faces + 3 * (size_t)(p.l.tbase[blockIdx.x] + tpre);
    for (int j = 0; j < 3 * ntri; ++j) {
        const int e = sh.table[idx * kTableWidth + j];
        const int o = edge_offset(e), k = edge_axis(e);
        const int xv = x + (o & 1), yv = y + ((o >> 1) & 1), zv = z + (o >> 2);
        const size_t gv = (size_t)sh.nb[nb_at(xv, yv, zv)] * kBlockVoxels + (xv & 7) + 8 * (yv & 7) + 64 * (zv & 7);
        const int bv = (int)(gv / kBlockVoxels);
        out[j] = (int)(p.l.vbase[bv] + p.l.vpre[gv] + __popc(p.l.info[gv] & ((1 << k) - 1)));
    }
}

int check_grid(const char *what, double s, int trunc) {
    static thread_local char msg[160];
    if (!(s > 0.0) || !(s < INFINITY)) {
        snprintf(msg, sizeof msg, "%s: voxel_size must be positive and finite", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    if (trunc < 1 || trunc > 4) {
        snprintf(msg, sizeof msg, "%s: trunc must be 1..4 voxels", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    return 0;
}

}  // namespace

extern "C" int64_t pmb200_tsdf_alloc_workspace_bytes(int64_t n_points) {
    if (n_points < 0 || n_points >= kMaxPoints) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc_workspace_bytes: 0 <= n < 2^28");
    Carver c{nullptr};
    AllocLayout l;
    if (!alloc_layout(c, n_points, l)) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc_workspace_bytes: no CUDA device to size the CUB sort for");
    return (int64_t)c.used;
}

extern "C" int pmb200_tsdf_alloc(const float *points, int64_t n_points, double voxel_size, int trunc, int64_t *n_blocks_out,
                                 void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!points && n_points > 0) || !n_blocks_out || !workspace) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc: null pointer");
    if (n_points < 0 || n_points >= kMaxPoints) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc: 0 <= n < 2^28");
    if (const int rc = check_grid("tsdf_alloc", voxel_size, trunc)) return rc;
    Carver c{static_cast<char *>(workspace)};
    AllocLayout l;
    if (!alloc_layout(c, n_points, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc: workspace smaller than tsdf_alloc_workspace_bytes(n)");
    *n_blocks_out = 0;
    if (n_points == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int m = (int)(8 * n_points);
    cudaMemsetAsync(l.n_unique, 0, 2 * sizeof(long long), st);
    alloc_keys_kernel<<<grid_blocks(n_points), kBlock, 0, st>>>(points, (int)n_points, voxel_size, trunc * voxel_size, l.keys_in, l.bad);
    size_t bytes = l.cub_bytes;
    if (cub::DeviceRadixSort::SortKeys(l.cub, bytes, l.keys_in, l.keys_sorted, m, 0, 63, st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_alloc (sort)");
    bytes = l.cub_bytes;
    if (cub::DeviceSelect::Unique(l.cub, bytes, l.keys_sorted, l.unique, l.n_unique, m, st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_alloc (unique)");
    long long host[2] = {0, 0};
    if (cudaMemcpyAsync(host, l.n_unique, sizeof host, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_alloc");
    if ((int)(host[1] & 0xffffffff) != 0)
        return pmb200_internal_fail(PMB200_EINVAL, "tsdf_alloc: a seed point is not finite or its voxel index does not fit in "
                                                   "[-2^23, 2^23) (use a larger voxel size)");
    *n_blocks_out = host[0];
    return pmb200_internal_launch_status("tsdf_alloc");
}

extern "C" int64_t pmb200_tsdf_integrate_workspace_bytes(int n_views) {
    if (n_views < 1) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate_workspace_bytes: n_views >= 1");
    return (int64_t)align256((size_t)n_views * sizeof(pmb200_tsdf_view));
}

extern "C" int pmb200_tsdf_integrate(const uint64_t *block_keys, int64_t n_blocks, double voxel_size, int trunc,
                                     const pmb200_tsdf_view *views_host, int n_views, const float *depth_flat,
                                     const float *image_flat, float *tsdf_out, float *weight_out, unsigned char *colour_out,
                                     void *workspace, int64_t workspace_bytes, void *stream) {
    if (!block_keys || !views_host || !depth_flat || !image_flat || !tsdf_out || !weight_out || !colour_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate: null pointer");
    if (n_blocks < 1 || n_blocks >= kMaxBlocks) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate: 1 <= n_blocks < 2^22");
    if (n_views < 1) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate: n_views >= 1");
    if (const int rc = check_grid("tsdf_integrate", voxel_size, trunc)) return rc;
    for (int v = 0; v < n_views; ++v)
        if (views_host[v].height < 1 || views_host[v].width < 1 || (long long)views_host[v].height * views_host[v].width >= (1ll << 31))
            return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate: every view needs 1 <= H, W and H * W < 2^31");
    const size_t table = (size_t)n_views * sizeof(pmb200_tsdf_view);
    if (workspace_bytes < (int64_t)table) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_integrate: workspace smaller than tsdf_integrate_workspace_bytes(n_views)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (cudaMemcpyAsync(workspace, views_host, table, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_integrate (view table)");
    IntegrateParams p;
    p.keys = reinterpret_cast<const unsigned long long *>(block_keys);
    p.views = static_cast<const pmb200_tsdf_view *>(workspace);
    p.n_views = n_views;
    p.s = voxel_size;
    p.tau = trunc * voxel_size;
    p.depth = depth_flat;
    p.image = image_flat;
    p.tsdf = tsdf_out;
    p.weight = weight_out;
    p.colour = reinterpret_cast<uchar4 *>(colour_out);
    integrate_kernel<<<(unsigned)n_blocks, kVoxThreads, 0, st>>>(p);
    return pmb200_internal_launch_status("tsdf_integrate");
}

extern "C" int64_t pmb200_tsdf_mesh_workspace_bytes(int64_t n_blocks) {
    if (n_blocks < 1 || n_blocks >= kMaxBlocks) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_mesh_workspace_bytes: 1 <= n_blocks < 2^22");
    Carver c{nullptr};
    MeshLayout l;
    if (!mesh_layout(c, n_blocks, l)) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_mesh_workspace_bytes: no CUDA device to size the CUB scan for");
    return (int64_t)c.used;
}

namespace {

int mesh_params(const char *what, const uint64_t *block_keys, int64_t n_blocks, double s, const float *tsdf, const float *weight,
                int min_weight, void *workspace, int64_t workspace_bytes, MeshParams &p) {
    static thread_local char msg[160];
    if (!block_keys || !tsdf || !weight || !workspace) {
        snprintf(msg, sizeof msg, "%s: null pointer", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    if (n_blocks < 1 || n_blocks >= kMaxBlocks) {
        snprintf(msg, sizeof msg, "%s: 1 <= n_blocks < 2^22", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    if (min_weight < 1) {
        snprintf(msg, sizeof msg, "%s: min_weight >= 1", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    if (!(s > 0.0) || !(s < INFINITY)) {
        snprintf(msg, sizeof msg, "%s: voxel_size must be positive and finite", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    Carver c{static_cast<char *>(workspace)};
    if (!mesh_layout(c, n_blocks, p.l) || workspace_bytes < (int64_t)c.used) {
        snprintf(msg, sizeof msg, "%s: workspace smaller than tsdf_mesh_workspace_bytes(n_blocks)", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    p.keys = reinterpret_cast<const unsigned long long *>(block_keys);
    p.n_blocks = (int)n_blocks;
    p.tsdf = tsdf;
    p.weight = weight;
    p.colour = nullptr;
    p.min_weight = (float)min_weight;
    p.s = s;
    p.verts = nullptr;
    p.faces = nullptr;
    return 0;
}

}  // namespace

extern "C" int pmb200_tsdf_mesh_count(const uint64_t *block_keys, int64_t n_blocks, const float *tsdf, const float *weight, int min_weight,
                                      int64_t *totals_out, void *workspace, int64_t workspace_bytes, void *stream) {
    MeshParams p;
    if (!totals_out) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_mesh_count: null pointer");
    if (const int rc = mesh_params("tsdf_mesh_count", block_keys, n_blocks, 1.0, tsdf, weight, min_weight, workspace, workspace_bytes, p))
        return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int nb = (int)n_blocks;
    mesh_count_kernel<<<nb, kVoxThreads, 0, st>>>(p);
    cudaMemsetAsync(p.l.vbase, 0, sizeof(long long), st);
    cudaMemsetAsync(p.l.tbase, 0, sizeof(long long), st);
    size_t bytes = p.l.cub_bytes;
    if (cub::DeviceScan::InclusiveSum(p.l.cub, bytes, p.l.bcount, p.l.vbase + 1, nb, st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_mesh_count (scan)");
    bytes = p.l.cub_bytes;
    if (cub::DeviceScan::InclusiveSum(p.l.cub, bytes, p.l.bcount + nb, p.l.tbase + 1, nb, st) != cudaSuccess)
        return pmb200_internal_launch_status("tsdf_mesh_count (scan)");
    cudaMemcpyAsync(totals_out, p.l.vbase + nb, sizeof(int64_t), cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(totals_out + 1, p.l.tbase + nb, sizeof(int64_t), cudaMemcpyDeviceToDevice, st);
    return pmb200_internal_launch_status("tsdf_mesh_count");
}

extern "C" int pmb200_tsdf_mesh_write(const uint64_t *block_keys, int64_t n_blocks, double voxel_size, const float *tsdf,
                                      const float *weight, const unsigned char *colour, int min_weight, unsigned char *vertices_out,
                                      int *faces_out, void *workspace, int64_t workspace_bytes, void *stream) {
    MeshParams p;
    if (!colour || !vertices_out || !faces_out) return pmb200_internal_fail(PMB200_EINVAL, "tsdf_mesh_write: null pointer");
    if (const int rc = mesh_params("tsdf_mesh_write", block_keys, n_blocks, voxel_size, tsdf, weight, min_weight, workspace,
                                   workspace_bytes, p))
        return rc;
    p.colour = reinterpret_cast<const uchar4 *>(colour);
    p.verts = vertices_out;
    p.faces = faces_out;
    mesh_write_kernel<<<(int)n_blocks, kVoxThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return pmb200_internal_launch_status("tsdf_mesh_write");
}
