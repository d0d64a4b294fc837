// pm_cloud.cu -- point-cloud thinning and exact nearest-neighbour distances for the DTU point-cloud evaluation
// (reference evaluations/dtu: reducePts_haa.m, MaxDistCP.m; semantics restated in INTEGRATION.md "DTU evaluation"), and the
// polygon crop, voxel down-sampling and ICP correspondences of the Tanks and Temples evaluation (INTEGRATION.md "Tanks and
// Temples evaluation"; definitions in include/patchmatch_b200.h).
//
// The searches sit on one spatial structure over a float64 cloud:
//   - fine cells of edge `cell`; fine coordinate f = floor(x / cell), clamped to [-2^20, 2^20);
//   - coarse cells of 16^3 fine cells (coarse coordinate f >> 4, 17 bits per axis);
//   - a 63-bit key  coarse(x,y,z) << 12 | fine-within-coarse(x,y,z): sorting the points by it (CUB radix sort) makes every
//     fine cell AND every coarse cell a contiguous run of the sorted cloud;
//   - two open-addressing hash tables (key -> [start, end) of the run), capacity the power of two >= 2 n: memory is O(n),
//     independent of the extent of the cloud.
// Clamping is monotone and never increases a cell distance, so "every point within r is in the neighbouring cells" and
// "a point k cells away is at least (k - 1) cells away" stay true for clamped points; they only make far-out cells crowded.
// Every distance is float64, ((dx*dx + dy*dy) + dz*dz) with no fused multiply-add, the order numpy evaluates it in.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kBlock = 256;
constexpr int kFineBits = 4;                        // 16 fine cells per coarse cell and axis
constexpr long long kFineClamp = 1ll << 20;         // fine coordinates in [-2^20, 2^20)
constexpr long long kCoarseBias = 1ll << 16;        // coarse coordinates (17 bits) biased to be non-negative
constexpr unsigned long long kEmpty = ~0ull;        // keys use 63 bits: never equal to kEmpty
constexpr int kThinMaxRounds = 256;                 // bound of the thinning rounds (one launch each)
constexpr int kFineRings = 2;                       // nearest search: fine Chebyshev rings before the coarse level takes over
constexpr double kMaxCellsPerDist = 256.0;         // nearest search: cell >= max_dist / 256, so at most 17 coarse rings
constexpr double kCellSlack = 1e-6;                 // relative margin for the rounding of floor(x / cell)
constexpr unsigned char kUndecided = 0, kAccepted = 1, kRejected = 2;

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

inline long long table_capacity(long long n) {
    long long c = 1;
    while (c < 2 * n) c <<= 1;
    return c < 2 ? 2 : c;
}

__device__ inline double dist2(double ax, double ay, double az, double bx, double by, double bz) {
    const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ inline int fine_coord(double x, double inv_cell) {
    const double f = floor(x * inv_cell);
    // NaN and anything beyond the range land on the clamp (a NaN coordinate never passes a distance test anyway)
    return (int)fmin(fmax(f, (double)-kFineClamp), (double)(kFineClamp - 1));
}

__device__ inline unsigned long long coarse_key(int cx, int cy, int cz) {
    return ((unsigned long long)(cx + kCoarseBias) << 34) | ((unsigned long long)(cy + kCoarseBias) << 17) |
           (unsigned long long)(cz + kCoarseBias);
}

__device__ inline unsigned long long fine_key(int fx, int fy, int fz) {
    const unsigned long long c = coarse_key(fx >> kFineBits, fy >> kFineBits, fz >> kFineBits);
    const int m = (1 << kFineBits) - 1;
    return (c << (3 * kFineBits)) | ((unsigned long long)(fx & m) << (2 * kFineBits)) |
           ((unsigned long long)(fy & m) << kFineBits) | (unsigned long long)(fz & m);
}

__device__ inline unsigned hash_slot(unsigned long long key, unsigned long long mask) {
    return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 20) & (unsigned)mask;
}

struct Table {
    unsigned long long *keys;
    int *start, *end;
    unsigned long long mask;  // capacity - 1
};

// [start, end) of the run with this key, or start == end when there is none
__device__ inline int2 table_find(const Table &t, unsigned long long key) {
    unsigned s = hash_slot(key, t.mask);
    while (true) {
        const unsigned long long k = __ldg(t.keys + s);
        if (k == key) return make_int2(__ldg(t.start + s), __ldg(t.end + s));
        if (k == kEmpty) return make_int2(0, 0);
        s = (s + 1) & (unsigned)t.mask;
    }
}

__device__ inline unsigned table_insert(const Table &t, unsigned long long key) {
    unsigned s = hash_slot(key, t.mask);
    while (true) {
        const unsigned long long prev = atomicCAS(t.keys + s, kEmpty, key);
        if (prev == kEmpty || prev == key) return s;
        s = (s + 1) & (unsigned)t.mask;
    }
}

// ---- grid build: keys -> radix sort -> sorted coordinates -> run tables ----------------------------------------------------

struct Grid {
    unsigned long long *keys_in, *keys_sorted;
    int *idx_in, *idx_sorted;
    double *pts;  // [n][3] in key order
    Table fine, coarse;
    void *cub_temp;
    size_t cub_bytes;
};

__global__ void __launch_bounds__(kBlock) grid_keys_kernel(const double *p, int n, double inv_cell, unsigned long long *keys, int *idx) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        keys[i] = fine_key(fine_coord(p[3 * (size_t)i], inv_cell), fine_coord(p[3 * (size_t)i + 1], inv_cell), fine_coord(p[3 * (size_t)i + 2], inv_cell));
        idx[i] = i;
    }
}

__global__ void __launch_bounds__(kBlock) grid_gather_kernel(const double *p, int n, const int *idx, double *out) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const int j = idx[i];
        out[3 * (size_t)i] = p[3 * (size_t)j]; out[3 * (size_t)i + 1] = p[3 * (size_t)j + 1]; out[3 * (size_t)i + 2] = p[3 * (size_t)j + 2];
    }
}

// run boundaries of `keys >> shift`: the first element of a run inserts the key and its start, the last one its end
__global__ void __launch_bounds__(kBlock) grid_table_kernel(const unsigned long long *keys, int n, int shift, Table t) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const unsigned long long k = keys[i] >> shift;
        const bool first = i == 0 || (keys[i - 1] >> shift) != k;
        const bool last = i == n - 1 || (keys[i + 1] >> shift) != k;
        if (!first && !last) continue;
        const unsigned s = table_insert(t, k);
        if (first) t.start[s] = i;
        if (last) t.end[s] = i + 1;
    }
}

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

// Lays out a grid over n points.  Returns false when CUB cannot size its temporary storage.
bool carve_grid(Carver &c, long long n, bool with_coarse, Grid &g) {
    const long long cap = table_capacity(n);
    g.keys_in = c.take<unsigned long long>(n);
    g.keys_sorted = c.take<unsigned long long>(n);
    g.idx_in = c.take<int>(n);
    g.idx_sorted = c.take<int>(n);
    g.pts = c.take<double>(3 * n);
    g.fine.keys = c.take<unsigned long long>(cap);
    g.fine.start = c.take<int>(cap);
    g.fine.end = c.take<int>(cap);
    g.fine.mask = (unsigned long long)(cap - 1);
    if (with_coarse) {
        g.coarse.keys = c.take<unsigned long long>(cap);
        g.coarse.start = c.take<int>(cap);
        g.coarse.end = c.take<int>(cap);
    } else {
        g.coarse.keys = nullptr; g.coarse.start = g.coarse.end = nullptr;
    }
    g.coarse.mask = (unsigned long long)(cap - 1);
    size_t bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int *)nullptr,
                                        (int *)nullptr, (int)(n < 1 ? 1 : n), 0, 63) != cudaSuccess)
        return false;
    g.cub_bytes = bytes;
    g.cub_temp = c.take<char>(bytes);
    return true;
}

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 ? 65535 : b));
}

cudaError_t build_grid(const Grid &g, const double *points, int n, double cell, bool with_coarse, cudaStream_t st) {
    const int blocks = grid_blocks(n);
    const size_t cap = (size_t)g.fine.mask + 1;
    cudaMemsetAsync(g.fine.keys, 0xff, cap * sizeof(unsigned long long), st);
    if (with_coarse) cudaMemsetAsync(g.coarse.keys, 0xff, cap * sizeof(unsigned long long), st);
    grid_keys_kernel<<<blocks, kBlock, 0, st>>>(points, n, 1.0 / cell, g.keys_in, g.idx_in);
    size_t bytes = g.cub_bytes;
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(g.cub_temp, bytes, g.keys_in, g.keys_sorted, g.idx_in, g.idx_sorted, n, 0, 63, st);
    if (e != cudaSuccess) return e;
    grid_gather_kernel<<<blocks, kBlock, 0, st>>>(points, n, g.idx_sorted, g.pts);
    grid_table_kernel<<<blocks, kBlock, 0, st>>>(g.keys_sorted, n, 0, g.fine);
    if (with_coarse) grid_table_kernel<<<blocks, kBlock, 0, st>>>(g.keys_sorted, n, 3 * kFineBits, g.coarse);
    return cudaSuccess;
}

// ---- thinning: lexicographically-first maximal independent set of "distance <= dst" in rank order ------------------------
// A point is accepted once every earlier (lower-rank) neighbour is rejected, rejected as soon as one earlier neighbour is
// accepted.  Decisions are final and correct when made, so a round may read its own round's decisions (they only speed it up).
// One round per launch; round r does nothing once round r-1 left no point undecided, so the host enqueues kThinMaxRounds
// launches without ever waiting.  A cloud still undecided after the last round is reported, not looped on.

struct ThinParams {
    const double *pts;        // sorted
    const int *rank;          // sorted
    unsigned char *state;     // sorted
    Table fine;
    double inv_cell, dst;
    int n;
    int *pending;             // [kThinMaxRounds]: 1 when some point was still undecided after that round
};

__global__ void __launch_bounds__(kBlock) thin_rank_kernel(const int *rank, const int *idx_sorted, int n, int *rank_sorted,
                                                           unsigned char *state) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        rank_sorted[i] = rank[idx_sorted[i]];
        state[i] = kUndecided;
    }
}

__global__ void __launch_bounds__(kBlock) thin_round_kernel(const ThinParams p, int round) {
    if (round > 0 && *(volatile int *)(p.pending + round - 1) == 0) return;
    bool left = false;
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < p.n; i += gridDim.x * kBlock) {
        if (((volatile unsigned char *)p.state)[i] != kUndecided) continue;
        const double x = p.pts[3 * (size_t)i], y = p.pts[3 * (size_t)i + 1], z = p.pts[3 * (size_t)i + 2];
        const int ri = p.rank[i];
        const int fx = fine_coord(x, p.inv_cell), fy = fine_coord(y, p.inv_cell), fz = fine_coord(z, p.inv_cell);
        bool blocked = false, rejected = false;
        for (int dx = -1; dx <= 1 && !rejected; ++dx)
            for (int dy = -1; dy <= 1 && !rejected; ++dy)
                for (int dz = -1; dz <= 1 && !rejected; ++dz) {
                    const long long cx = (long long)fx + dx, cy = (long long)fy + dy, cz = (long long)fz + dz;
                    if (cx < -kFineClamp || cx >= kFineClamp || cy < -kFineClamp || cy >= kFineClamp || cz < -kFineClamp || cz >= kFineClamp)
                        continue;
                    const int2 r = table_find(p.fine, fine_key((int)cx, (int)cy, (int)cz));
                    for (int j = r.x; j < r.y; ++j) {
                        if (__ldg(p.rank + j) >= ri) continue;
                        const double d2 = dist2(x, y, z, __ldg(p.pts + 3 * (size_t)j), __ldg(p.pts + 3 * (size_t)j + 1), __ldg(p.pts + 3 * (size_t)j + 2));
                        if (!(__dsqrt_rn(d2) <= p.dst)) continue;
                        const unsigned char s = ((volatile unsigned char *)p.state)[j];
                        if (s == kAccepted) { rejected = true; break; }
                        if (s == kUndecided) blocked = true;
                    }
                }
        if (rejected) p.state[i] = kRejected;
        else if (!blocked) p.state[i] = kAccepted;
        else left = true;
    }
    if (__syncthreads_or(left) && threadIdx.x == 0) p.pending[round] = 1;
}

__global__ void __launch_bounds__(kBlock) thin_scatter_kernel(const unsigned char *state, const int *idx_sorted, int n,
                                                              const int *pending, unsigned char *keep, int *undecided) {
    const bool unfinished = pending[kThinMaxRounds - 1] != 0;
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const unsigned char s = state[i];
        keep[idx_sorted[i]] = s == kAccepted ? 1 : 0;
        if (unfinished && s == kUndecided) atomicAdd(undecided, 1);
    }
}

// ---- nearest distance, capped, with or without the block membership of MaxDistCP--------------------------------------------

struct NearestParams {
    const double *from;
    int n_from;
    Table fine, coarse;
    const double *pts;        // "to" cloud, sorted
    double inv_cell, cell, max_dist;
    double bb_lo[3], range[3];  // range: MaxDistCP's last block index per axis
    bool blocks;                // false: every query is searched (no block membership)
    double *out;
};

// MaxDistCP's blocks along one axis: Low = BB_lo + k * MaxDist, High = Low + MaxDist, k = 0 .. floor((BB_hi - BB_lo) / MaxDist),
// tested with the same float64 expressions (adjacent blocks may overlap or leave a gap of one rounding step; both are kept).
// `range` = floor((BB_hi - BB_lo) / MaxDist) comes from the host; k0 is only a first guess (the exact tests decide).
__device__ inline bool in_some_block(double q, double lo, double range, double m, double inv_m) {
    if (!(range >= 0.0)) return false;
    const double k0 = floor((q - lo) * inv_m);
    if (!(k0 >= -1.0 && k0 <= range + 1.0)) return false;  // far outside (or not finite): also keeps k0 +- 1 exact
    for (double k = k0 - 1.0; k <= k0 + 1.0; k += 1.0) {
        if (k < 0.0 || k > range) continue;
        const double low = __dadd_rn(lo, __dmul_rn(k, m)), high = __dadd_rn(low, m);  // no fused multiply-add
        if (q >= low && q < high) return true;
    }
    return false;
}

__device__ inline void scan_run(const double *pts, int2 r, double x, double y, double z, double &best) {
    for (int j = r.x; j < r.y; ++j) {
        const double d2 = dist2(x, y, z, __ldg(pts + 3 * (size_t)j), __ldg(pts + 3 * (size_t)j + 1), __ldg(pts + 3 * (size_t)j + 2));
        best = fmin(best, d2);
    }
}

__device__ inline bool in_range(long long c, long long lo, long long hi) { return c >= lo && c < hi; }

__global__ void __launch_bounds__(kBlock) nearest_kernel(const NearestParams p) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < p.n_from; i += gridDim.x * kBlock) {
        const double x = p.from[3 * (size_t)i], y = p.from[3 * (size_t)i + 1], z = p.from[3 * (size_t)i + 2];
        const double m = p.max_dist, inv_m = 1.0 / p.max_dist;
        if (p.blocks && !(in_some_block(x, p.bb_lo[0], p.range[0], m, inv_m) && in_some_block(y, p.bb_lo[1], p.range[1], m, inv_m) &&
                          in_some_block(z, p.bb_lo[2], p.range[2], m, inv_m))) {
            p.out[i] = p.max_dist;
            continue;
        }
        double best = INFINITY;  // squared
        bool done = false;
        const int fx = fine_coord(x, p.inv_cell), fy = fine_coord(y, p.inv_cell), fz = fine_coord(z, p.inv_cell);
        // fine level: Chebyshev rings 0..kFineRings; after ring k every unvisited point is >= k cells away
        for (int k = 0; k <= kFineRings && !done; ++k) {
            for (int dx = -k; dx <= k; ++dx)
                for (int dy = -k; dy <= k; ++dy) {
                    const bool face = dx == -k || dx == k || dy == -k || dy == k;
                    for (int dz = -k; dz <= k; dz += face ? 1 : (2 * k > 0 ? 2 * k : 1)) {
                        const long long cx = (long long)fx + dx, cy = (long long)fy + dy, cz = (long long)fz + dz;
                        if (!in_range(cx, -kFineClamp, kFineClamp) || !in_range(cy, -kFineClamp, kFineClamp) || !in_range(cz, -kFineClamp, kFineClamp))
                            continue;
                        scan_run(p.pts, table_find(p.fine, fine_key((int)cx, (int)cy, (int)cz)), x, y, z, best);
                    }
                }
            const double reach = (k - kCellSlack) * p.cell;
            if (k > 0 && (__dsqrt_rn(best) <= reach || reach >= p.max_dist)) done = true;
        }
        if (!done) {
            // coarse level: rings of coarse cells, a run scanned only when its per-axis cell distance could beat the best
            const int cx0 = fx >> kFineBits, cy0 = fy >> kFineBits, cz0 = fz >> kFineBits;
            const double coarse = p.cell * (1 << kFineBits);
            const long long clo = -(kFineClamp >> kFineBits), chi = kFineClamp >> kFineBits;
            for (int m = 0; !done; ++m) {
                for (int dx = -m; dx <= m; ++dx)
                    for (int dy = -m; dy <= m; ++dy) {
                        const bool face = dx == -m || dx == m || dy == -m || dy == m;
                        for (int dz = -m; dz <= m; dz += face ? 1 : (2 * m > 0 ? 2 * m : 1)) {
                            const long long cx = (long long)cx0 + dx, cy = (long long)cy0 + dy, cz = (long long)cz0 + dz;
                            if (!in_range(cx, clo, chi) || !in_range(cy, clo, chi) || !in_range(cz, clo, chi)) continue;
                            const double gx = fmax(abs(dx) - 1 - kCellSlack, 0.0) * coarse, gy = fmax(abs(dy) - 1 - kCellSlack, 0.0) * coarse,
                                         gz = fmax(abs(dz) - 1 - kCellSlack, 0.0) * coarse;
                            if (gx * gx + gy * gy + gz * gz > best) continue;
                            scan_run(p.pts, table_find(p.coarse, coarse_key((int)cx, (int)cy, (int)cz)), x, y, z, best);
                        }
                    }
                const double reach = (m - kCellSlack) * coarse;
                if (m > 0 && (__dsqrt_rn(best) <= reach || reach >= p.max_dist)) done = true;
            }
        }
        p.out[i] = fmin(__dsqrt_rn(best), p.max_dist);
    }
}

__global__ void __launch_bounds__(kBlock) fill_kernel(double *out, int n, double v) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) out[i] = v;
}

long long thin_layout(Carver &c, long long n, Grid &g, int *&rank_sorted, unsigned char *&state, int *&pending) {
    if (!carve_grid(c, n, false, g)) return -1;
    rank_sorted = c.take<int>(n);
    state = c.take<unsigned char>(n);
    pending = c.take<int>(kThinMaxRounds);
    return (long long)c.used;
}

long long nearest_layout(Carver &c, long long n_to, Grid &g) {
    if (!carve_grid(c, n_to, true, g)) return -1;
    return (long long)c.used;
}

// ---- Tanks and Temples evaluation: polygon crop, voxel down-sampling, ICP correspondences (include/patchmatch_b200.h) ----

constexpr int kMaxPolygon = 128;  // crop polygon vertices held in the kernel parameters
constexpr int kMoments = 18;      // ICP query: count, sum d^2, sum p, sum q, sum q p^T, sum |p|^2

struct Affine {
    double m[12];  // rows of the top 3 x 4 of a 4 x 4 whose last row is 0 0 0 1
};

// ((m0 x + m1 y) + m2 z) + m3 per row, every operation rounded on its own (no fused multiply-add)
__device__ inline void apply_affine(const Affine &t, double x, double y, double z, double &ox, double &oy, double &oz) {
    ox = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(t.m[0], x), __dmul_rn(t.m[1], y)), __dmul_rn(t.m[2], z)), t.m[3]);
    oy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(t.m[4], x), __dmul_rn(t.m[5], y)), __dmul_rn(t.m[6], z)), t.m[7]);
    oz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(t.m[8], x), __dmul_rn(t.m[9], y)), __dmul_rn(t.m[10], z)), t.m[11]);
}

__device__ inline double pick(int a, double x, double y, double z) { return a == 0 ? x : (a == 1 ? y : z); }

struct CropParams {
    Affine t;
    int u, v, w, nv;
    double axis_min, axis_max;
    double pu[kMaxPolygon], pv[kMaxPolygon];
};

__global__ void __launch_bounds__(kBlock) crop_kernel(const double *p, int n, const CropParams c, double *out, unsigned char *keep) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        double x, y, z;
        apply_affine(c.t, p[3 * (size_t)i], p[3 * (size_t)i + 1], p[3 * (size_t)i + 2], x, y, z);
        out[3 * (size_t)i] = x; out[3 * (size_t)i + 1] = y; out[3 * (size_t)i + 2] = z;
        const double pw = pick(c.w, x, y, z), pu = pick(c.u, x, y, z), pv = pick(c.v, x, y, z);
        bool inside = false;
        if (pw >= c.axis_min && pw <= c.axis_max) {
            for (int a = 0; a < c.nv; ++a) {
                const int b = a + 1 == c.nv ? 0 : a + 1;
                const double va = c.pv[a], vb = c.pv[b];
                if ((va < pv && vb >= pv) || (vb < pv && va >= pv)) {
                    const double cross = __dadd_rn(c.pu[a], __dmul_rn(__ddiv_rn(__dsub_rn(pv, va), __dsub_rn(vb, va)), __dsub_rn(c.pu[b], c.pu[a])));
                    if (cross < pu) inside = !inside;
                }
            }
        }
        keep[i] = inside ? 1 : 0;
    }
}

struct VoxelParams {
    double origin[3], size;
    int bits[3];  // key bits per axis (bits of the largest index)
    bool split;   // the x index does not fit beside y and z in 64 bits: sort by (y, z), then stably by x
};

__device__ inline int voxel_index(double x, double origin, double size) { return (int)floor(__ddiv_rn(__dsub_rn(x, origin), size)); }

__device__ inline int3 voxel_of(const double *p, int i, const VoxelParams &v) {
    return make_int3(voxel_index(p[3 * (size_t)i], v.origin[0], v.size), voxel_index(p[3 * (size_t)i + 1], v.origin[1], v.size),
                     voxel_index(p[3 * (size_t)i + 2], v.origin[2], v.size));
}

__global__ void __launch_bounds__(kBlock) voxel_keys_kernel(const double *p, int n, const VoxelParams v, unsigned long long *keys, int *idx) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const int3 c = voxel_of(p, i, v);
        const unsigned long long yz = ((unsigned long long)c.y << v.bits[2]) | (unsigned long long)c.z;
        keys[i] = v.split ? yz : (((unsigned long long)c.x << (v.bits[1] + v.bits[2])) | yz);
        idx[i] = i;
    }
}

__global__ void __launch_bounds__(kBlock) voxel_xkeys_kernel(const double *p, int n, const VoxelParams v, const int *idx, unsigned *xkeys) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock)
        xkeys[i] = (unsigned)voxel_index(p[3 * (size_t)idx[i]], v.origin[0], v.size);
}

__global__ void __launch_bounds__(kBlock) voxel_flags_kernel(const double *p, int n, const VoxelParams v, const int *idx, int *flags) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        bool first = i == 0;
        if (!first) {
            const int3 a = voxel_of(p, idx[i], v), b = voxel_of(p, idx[i - 1], v);
            first = a.x != b.x || a.y != b.y || a.z != b.z;
        }
        flags[i] = first ? 1 : 0;
    }
}

// runs[k] = sorted position where voxel k starts (k < count), runs[count] = n; *count_out = count
__global__ void __launch_bounds__(kBlock) voxel_runs_kernel(const int *flags, const int *pos, int n, int *runs, long long *count_out) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        if (flags[i]) runs[pos[i] - 1] = i;
        if (i == n - 1) { runs[pos[i]] = n; *count_out = pos[i]; }
    }
}

// one thread per voxel: the float64 sum of its points in sorted order (voxel, then original index), divided by their count
__global__ void __launch_bounds__(kBlock) voxel_mean_kernel(const double *p, const int *idx, const int *runs, const long long *count,
                                                            double *out) {
    const int nv = (int)*count;
    for (int k = blockIdx.x * kBlock + threadIdx.x; k < nv; k += gridDim.x * kBlock) {
        const int s = runs[k], e = runs[k + 1];
        double sx = 0.0, sy = 0.0, sz = 0.0;
        for (int j = s; j < e; ++j) {
            const int q = idx[j];
            sx = __dadd_rn(sx, p[3 * (size_t)q]); sy = __dadd_rn(sy, p[3 * (size_t)q + 1]); sz = __dadd_rn(sz, p[3 * (size_t)q + 2]);
        }
        const double c = (double)(e - s);
        out[3 * (size_t)k] = __ddiv_rn(sx, c); out[3 * (size_t)k + 1] = __ddiv_rn(sy, c); out[3 * (size_t)k + 2] = __ddiv_rn(sz, c);
    }
}

struct VoxelWork {
    unsigned long long *keys_in, *keys_sorted;
    unsigned *x_in, *x_sorted;
    int *idx_in, *idx_sorted, *flags, *pos, *runs;
    void *cub_temp;
    size_t cub_bytes;
};

long long voxel_layout(Carver &c, long long n, VoxelWork &w) {
    const int m = (int)(n < 1 ? 1 : n);
    w.keys_in = c.take<unsigned long long>(n);
    w.keys_sorted = c.take<unsigned long long>(n);
    w.x_in = c.take<unsigned>(n);
    w.x_sorted = c.take<unsigned>(n);
    w.idx_in = c.take<int>(n);
    w.idx_sorted = c.take<int>(n);
    w.flags = c.take<int>(n);
    w.pos = c.take<int>(n);
    w.runs = c.take<int>(n + 1);
    size_t a = 0, b = 0, s = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, a, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr, m, 0, 64) != cudaSuccess ||
        cub::DeviceRadixSort::SortPairs(nullptr, b, (unsigned *)nullptr, (unsigned *)nullptr, (int *)nullptr, (int *)nullptr, m, 0, 32) != cudaSuccess ||
        cub::DeviceScan::InclusiveSum(nullptr, s, (int *)nullptr, (int *)nullptr, m) != cudaSuccess)
        return -1;
    w.cub_bytes = a > b ? a : b;
    if (s > w.cub_bytes) w.cub_bytes = s;
    w.cub_temp = c.take<char>(w.cub_bytes);
    return (long long)c.used;
}

inline int bit_width(long long v) {
    int b = 0;
    while (b < 63 && (v >> b) != 0) ++b;
    return b;
}

// ---- ICP correspondences: nearest target point within max_dist, ties to the smallest target index ----------------------

struct IcpParams {
    const double *src;
    int n_src;
    Affine t;
    Table fine, coarse;
    const double *pts;   // target, sorted
    const int *idx;      // target, sorted -> original index
    double inv_cell, cell, max_dist, origin[3];
    int *corr;           // [n_src] or NULL
    double *partials;    // [gridDim.x][kMoments]
};

__device__ inline void scan_run_index(const double *pts, const int *idx, int2 r, double x, double y, double z, double &best, int &bi, int &bj) {
    for (int j = r.x; j < r.y; ++j) {
        const double d2 = dist2(x, y, z, __ldg(pts + 3 * (size_t)j), __ldg(pts + 3 * (size_t)j + 1), __ldg(pts + 3 * (size_t)j + 2));
        const int id = __ldg(idx + j);
        if (d2 < best || (d2 == best && id < bi)) { best = d2; bi = id; bj = j; }
    }
}

// The ring search of nearest_kernel, keeping the index: after fine ring k every unvisited point is more than
// (k - kCellSlack) cells away, so a point at exactly the best distance is never left unvisited and the tie rule is exact.
__device__ inline int nearest_index(const IcpParams &p, double x, double y, double z, double &best) {
    best = INFINITY;
    int bi = 0x7fffffff, bj = -1;
    bool done = false;
    const int fx = fine_coord(x, p.inv_cell), fy = fine_coord(y, p.inv_cell), fz = fine_coord(z, p.inv_cell);
    for (int k = 0; k <= kFineRings && !done; ++k) {
        for (int dx = -k; dx <= k; ++dx)
            for (int dy = -k; dy <= k; ++dy) {
                const bool face = dx == -k || dx == k || dy == -k || dy == k;
                for (int dz = -k; dz <= k; dz += face ? 1 : (2 * k > 0 ? 2 * k : 1)) {
                    const long long cx = (long long)fx + dx, cy = (long long)fy + dy, cz = (long long)fz + dz;
                    if (!in_range(cx, -kFineClamp, kFineClamp) || !in_range(cy, -kFineClamp, kFineClamp) || !in_range(cz, -kFineClamp, kFineClamp))
                        continue;
                    scan_run_index(p.pts, p.idx, table_find(p.fine, fine_key((int)cx, (int)cy, (int)cz)), x, y, z, best, bi, bj);
                }
            }
        const double reach = (k - kCellSlack) * p.cell;
        if (k > 0 && (__dsqrt_rn(best) <= reach || reach >= p.max_dist)) done = true;
    }
    if (!done) {
        const int cx0 = fx >> kFineBits, cy0 = fy >> kFineBits, cz0 = fz >> kFineBits;
        const double coarse = p.cell * (1 << kFineBits);
        const long long clo = -(kFineClamp >> kFineBits), chi = kFineClamp >> kFineBits;
        for (int m = 0; !done; ++m) {
            for (int dx = -m; dx <= m; ++dx)
                for (int dy = -m; dy <= m; ++dy) {
                    const bool face = dx == -m || dx == m || dy == -m || dy == m;
                    for (int dz = -m; dz <= m; dz += face ? 1 : (2 * m > 0 ? 2 * m : 1)) {
                        const long long cx = (long long)cx0 + dx, cy = (long long)cy0 + dy, cz = (long long)cz0 + dz;
                        if (!in_range(cx, clo, chi) || !in_range(cy, clo, chi) || !in_range(cz, clo, chi)) continue;
                        const double gx = fmax(abs(dx) - 1 - kCellSlack, 0.0) * coarse, gy = fmax(abs(dy) - 1 - kCellSlack, 0.0) * coarse,
                                     gz = fmax(abs(dz) - 1 - kCellSlack, 0.0) * coarse;
                        if (gx * gx + gy * gy + gz * gz > best) continue;
                        scan_run_index(p.pts, p.idx, table_find(p.coarse, coarse_key((int)cx, (int)cy, (int)cz)), x, y, z, best, bi, bj);
                    }
                }
            const double reach = (m - kCellSlack) * coarse;
            if (m > 0 && (__dsqrt_rn(best) <= reach || reach >= p.max_dist)) done = true;
        }
    }
    return bj;
}

// Each thread keeps its running sums in its own column of shared memory (no registers held across the search); the block
// sum is a fixed tree over the 256 columns.  No atomics, so the partials (and the ordered final sum of icp_finish_kernel)
// are the same bits on every run.
__global__ void __launch_bounds__(kBlock) icp_query_kernel(const IcpParams p) {
    __shared__ double acc[kMoments][kBlock];
    const int t = threadIdx.x;
    for (int k = 0; k < kMoments; ++k) acc[k][t] = 0.0;
    for (int i = blockIdx.x * kBlock + t; i < p.n_src; i += gridDim.x * kBlock) {
        double x, y, z, best;
        apply_affine(p.t, p.src[3 * (size_t)i], p.src[3 * (size_t)i + 1], p.src[3 * (size_t)i + 2], x, y, z);
        const int j = nearest_index(p, x, y, z, best);
        const bool hit = j >= 0 && __dsqrt_rn(best) <= p.max_dist;
        if (p.corr) p.corr[i] = hit ? __ldg(p.idx + j) : -1;
        if (!hit) continue;
        const double pp[3] = {__dsub_rn(x, p.origin[0]), __dsub_rn(y, p.origin[1]), __dsub_rn(z, p.origin[2])};
        const double qq[3] = {__dsub_rn(__ldg(p.pts + 3 * (size_t)j), p.origin[0]), __dsub_rn(__ldg(p.pts + 3 * (size_t)j + 1), p.origin[1]),
                              __dsub_rn(__ldg(p.pts + 3 * (size_t)j + 2), p.origin[2])};
        acc[0][t] += 1.0;
        acc[1][t] = __dadd_rn(acc[1][t], best);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            acc[2 + a][t] = __dadd_rn(acc[2 + a][t], pp[a]);
            acc[5 + a][t] = __dadd_rn(acc[5 + a][t], qq[a]);
#pragma unroll
            for (int b = 0; b < 3; ++b) acc[8 + 3 * a + b][t] = __dadd_rn(acc[8 + 3 * a + b][t], __dmul_rn(qq[a], pp[b]));
        }
        acc[17][t] = __dadd_rn(acc[17][t], __dadd_rn(__dadd_rn(__dmul_rn(pp[0], pp[0]), __dmul_rn(pp[1], pp[1])), __dmul_rn(pp[2], pp[2])));
    }
    __syncthreads();
    for (int o = kBlock / 2; o > 0; o >>= 1) {
        if (t < o)
            for (int k = 0; k < kMoments; ++k) acc[k][t] = __dadd_rn(acc[k][t], acc[k][t + o]);
        __syncthreads();
    }
    if (t < kMoments) p.partials[(size_t)blockIdx.x * kMoments + t] = acc[t][0];
}

// one CTA: moment k = the sum over blocks b of partials[b][k], each thread summing a fixed stride of blocks in order, then
// the 256 thread sums in a fixed tree
__global__ void __launch_bounds__(kBlock) icp_finish_kernel(const double *partials, int blocks, double *out) {
    __shared__ double s[kBlock];
    for (int k = 0; k < kMoments; ++k) {
        double v = 0.0;
        for (int b = threadIdx.x; b < blocks; b += kBlock) v = __dadd_rn(v, partials[(size_t)b * kMoments + k]);
        s[threadIdx.x] = v;
        __syncthreads();
        for (int o = kBlock / 2; o > 0; o >>= 1) {
            if (threadIdx.x < o) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + o]);
            __syncthreads();
        }
        if (threadIdx.x == 0) out[k] = s[0];
        __syncthreads();
    }
}

long long icp_target_layout(Carver &c, long long n_tgt, Grid &g) {
    if (!carve_grid(c, n_tgt, true, g)) return -1;
    return (long long)c.used;
}

// host checks of a 4 x 4 row-major transform: finite, last row exactly 0 0 0 1
bool affine_from_host(const double *m, Affine &t) {
    for (int k = 0; k < 16; ++k)
        if (!(m[k] == m[k]) || m[k] == INFINITY || m[k] == -INFINITY) return false;
    if (m[12] != 0.0 || m[13] != 0.0 || m[14] != 0.0 || m[15] != 1.0) return false;
    for (int k = 0; k < 12; ++k) t.m[k] = m[k];
    return true;
}

}  // namespace

extern "C" int64_t pmb200_thin_points_workspace_bytes(int64_t n) {
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "thin_points_workspace_bytes: 0 <= n < 2^31");
    Carver c{nullptr};
    Grid g;
    int *rs, *pend;
    unsigned char *st;
    const long long b = thin_layout(c, n, g, rs, st, pend);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "thin_points_workspace_bytes: no CUDA device to size the CUB sort for") : b;
}

extern "C" int pmb200_thin_points(const double *points, const int *rank, int64_t n, double dst, unsigned char *keep_out,
                                  int *undecided_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if (((!points || !rank || !keep_out) && n > 0) || !undecided_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "thin_points: null pointer");
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "thin_points: 0 <= n < 2^31");
    if (!(dst > 0.0) || !(dst < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, "thin_points: dst must be positive and finite");
    Carver c{static_cast<char *>(workspace)};
    Grid g;
    int *rank_sorted, *pending;
    unsigned char *state;
    const long long need = thin_layout(c, n, g, rank_sorted, state, pending);
    if (need < 0 || workspace_bytes < need) return pmb200_internal_fail(PMB200_EINVAL, "thin_points: workspace smaller than thin_points_workspace_bytes(n)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaMemsetAsync(undecided_out, 0, sizeof(int), st);
    if (n == 0) return pmb200_internal_launch_status("thin_points");
    // cells a little wider than dst: two points within dst are never more than one cell apart, whatever floor() rounds to
    const double cell = dst * (1.0 + kCellSlack);
    const cudaError_t e = build_grid(g, points, (int)n, cell, false, st);
    if (e != cudaSuccess) return pmb200_internal_launch_status("thin_points (sort)");
    const int blocks = grid_blocks(n);
    thin_rank_kernel<<<blocks, kBlock, 0, st>>>(rank, g.idx_sorted, (int)n, rank_sorted, state);
    cudaMemsetAsync(pending, 0, kThinMaxRounds * sizeof(int), st);
    ThinParams p;
    p.pts = g.pts; p.rank = rank_sorted; p.state = state; p.fine = g.fine;
    p.inv_cell = 1.0 / cell; p.dst = dst; p.n = (int)n; p.pending = pending;
    // rounds after the last one with work return at once: a grid of a few CTAs per SM keeps those launches cheap
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int round_blocks = blocks < 8 * sms ? blocks : 8 * sms;
    for (int r = 0; r < kThinMaxRounds; ++r) thin_round_kernel<<<round_blocks, kBlock, 0, st>>>(p, r);
    thin_scatter_kernel<<<blocks, kBlock, 0, st>>>(state, g.idx_sorted, (int)n, pending, keep_out, undecided_out);
    return pmb200_internal_launch_status("thin_points");
}

extern "C" int64_t pmb200_nearest_distance_workspace_bytes(int64_t n_to) {
    if (n_to < 0 || n_to >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance_workspace_bytes: 0 <= n_to < 2^31");
    Carver c{nullptr};
    Grid g;
    const long long b = nearest_layout(c, n_to, g);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "nearest_distance_workspace_bytes: no CUDA device to size the CUB sort for") : b;
}

namespace {

// pmb200_nearest_distance (bb_host: MaxDistCP's blocks) and pmb200_nearest_distance_capped (bb_host NULL: no blocks)
int nearest_distance_call(const double *to_points, int64_t n_to, const double *from_points, int64_t n_from, const double *bb_host,
                          double max_dist, double cell, double *dist_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!to_points && n_to > 0) || ((!from_points || !dist_out) && n_from > 0) || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance: null pointer");
    if (n_to < 0 || n_to >= (1ll << 31) || n_from < 0 || n_from >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance: 0 <= n_to, n_from < 2^31");
    if (!(max_dist > 0.0) || !(max_dist < INFINITY) || !(cell >= max_dist / kMaxCellsPerDist) || !(cell < INFINITY))
        return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance: max_dist finite and positive, max_dist / 256 <= cell < inf");
    Carver c{static_cast<char *>(workspace)};
    Grid g;
    const long long need = nearest_layout(c, n_to, g);
    if (need < 0 || workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance: workspace smaller than nearest_distance_workspace_bytes(n_to)");
    if (n_from == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int blocks = grid_blocks(n_from);
    if (n_to == 0) {
        fill_kernel<<<blocks, kBlock, 0, st>>>(dist_out, (int)n_from, max_dist);
        return pmb200_internal_launch_status("nearest_distance");
    }
    const cudaError_t e = build_grid(g, to_points, (int)n_to, cell, true, st);
    if (e != cudaSuccess) return pmb200_internal_launch_status("nearest_distance (sort)");
    NearestParams p;
    p.from = from_points; p.n_from = (int)n_from; p.fine = g.fine; p.coarse = g.coarse; p.pts = g.pts;
    p.inv_cell = 1.0 / cell; p.cell = cell; p.max_dist = max_dist;
    p.blocks = bb_host != nullptr;
    for (int a = 0; a < 3; ++a) {
        p.bb_lo[a] = p.blocks ? bb_host[a] : 0.0;
        p.range[a] = p.blocks ? floor((bb_host[3 + a] - bb_host[a]) / max_dist) : 0.0;
    }
    p.out = dist_out;
    nearest_kernel<<<blocks, kBlock, 0, st>>>(p);
    return pmb200_internal_launch_status("nearest_distance");
}

}  // namespace

extern "C" int pmb200_nearest_distance(const double *to_points, int64_t n_to, const double *from_points, int64_t n_from,
                                       const double *bb_host, double max_dist, double cell, double *dist_out, void *workspace,
                                       int64_t workspace_bytes, void *stream) {
    if (!bb_host) return pmb200_internal_fail(PMB200_EINVAL, "nearest_distance: null pointer");
    return nearest_distance_call(to_points, n_to, from_points, n_from, bb_host, max_dist, cell, dist_out, workspace, workspace_bytes, stream);
}

extern "C" int pmb200_nearest_distance_capped(const double *to_points, int64_t n_to, const double *from_points, int64_t n_from,
                                              double max_dist, double cell, double *dist_out, void *workspace, int64_t workspace_bytes,
                                              void *stream) {
    return nearest_distance_call(to_points, n_to, from_points, n_from, nullptr, max_dist, cell, dist_out, workspace, workspace_bytes, stream);
}

extern "C" int pmb200_crop_polygon(const double *points, int64_t n, const double *transform_host, int orthogonal_axis, double axis_min,
                                   double axis_max, const double *polygon_host, int n_vertices, double *points_out,
                                   unsigned char *keep_out, void *stream) {
    if (((!points || !points_out || !keep_out) && n > 0) || !transform_host || !polygon_host)
        return pmb200_internal_fail(PMB200_EINVAL, "crop_polygon: null pointer");
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "crop_polygon: 0 <= n < 2^31");
    if (orthogonal_axis < 0 || orthogonal_axis > 2) return pmb200_internal_fail(PMB200_EINVAL, "crop_polygon: orthogonal_axis must be 0, 1 or 2");
    if (n_vertices < 0 || n_vertices > kMaxPolygon) return pmb200_internal_fail(PMB200_EINVAL, "crop_polygon: 0 <= n_vertices <= 128");
    CropParams c;
    if (!affine_from_host(transform_host, c.t))
        return pmb200_internal_fail(PMB200_EINVAL, "crop_polygon: the transform must be finite with last row 0 0 0 1");
    c.w = orthogonal_axis;
    c.u = orthogonal_axis == 0 ? 1 : 0;
    c.v = orthogonal_axis == 2 ? 1 : 2;
    c.nv = n_vertices;
    c.axis_min = axis_min; c.axis_max = axis_max;
    for (int k = 0; k < n_vertices; ++k) { c.pu[k] = polygon_host[3 * k + c.u]; c.pv[k] = polygon_host[3 * k + c.v]; }
    if (n == 0) return 0;
    crop_kernel<<<grid_blocks(n), kBlock, 0, reinterpret_cast<cudaStream_t>(stream)>>>(points, (int)n, c, points_out, keep_out);
    return pmb200_internal_launch_status("crop_polygon");
}

extern "C" int64_t pmb200_voxel_downsample_workspace_bytes(int64_t n) {
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample_workspace_bytes: 0 <= n < 2^31");
    Carver c{nullptr};
    VoxelWork w;
    const long long b = voxel_layout(c, n, w);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample_workspace_bytes: no CUDA device to size the CUB calls for") : b;
}

extern "C" int pmb200_voxel_downsample(const double *points, int64_t n, const double *bounds_host, double voxel_size, double *points_out,
                                       int64_t *count_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if (((!points || !points_out) && n > 0) || !bounds_host || !count_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: null pointer");
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: 0 <= n < 2^31");
    if (!(voxel_size > 0.0) || !(voxel_size < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: voxel_size must be positive and finite");
    VoxelParams v;
    v.size = voxel_size;
    v.split = false;
    int total = 0;
    for (int a = 0; a < 3; ++a) {
        const double lo = bounds_host[a], hi = bounds_host[3 + a];
        if (!(lo <= hi) || !(lo > -INFINITY) || !(hi < INFINITY))
            return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: bounds must be finite with min <= max");
        v.origin[a] = lo - voxel_size * 0.5;
        // Open3D's check: the voxel bounds' extent must stay within voxel_size * INT_MAX
        if (voxel_size * 2147483647.0 < (hi + voxel_size * 0.5) - v.origin[a])
            return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: voxel_size too small for the extent (int32 voxel index overflow)");
        const double top = floor((hi - v.origin[a]) / voxel_size);  // the largest index (the ops are monotone)
        if (!(top >= 0.0) || top > 2147483647.0)
            return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: voxel_size too small for the extent (int32 voxel index overflow)");
        v.bits[a] = bit_width((long long)top);
        total += v.bits[a];
    }
    v.split = total > 64;
    Carver c{static_cast<char *>(workspace)};
    VoxelWork w;
    const long long need = voxel_layout(c, n, w);
    if (need < 0 || workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "voxel_downsample: workspace smaller than voxel_downsample_workspace_bytes(n)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaMemsetAsync(count_out, 0, sizeof(int64_t), st);
    if (n == 0) return pmb200_internal_launch_status("voxel_downsample");
    const int blocks = grid_blocks(n);
    voxel_keys_kernel<<<blocks, kBlock, 0, st>>>(points, (int)n, v, w.keys_in, w.idx_in);
    size_t bytes = w.cub_bytes;
    const int key_bits = v.split ? v.bits[1] + v.bits[2] : total;
    if (cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, w.keys_in, w.keys_sorted, w.idx_in, w.idx_sorted, (int)n, 0,
                                        key_bits > 0 ? key_bits : 1, st) != cudaSuccess)
        return pmb200_internal_launch_status("voxel_downsample (sort)");
    const int *order = w.idx_sorted;
    if (v.split) {  // radix sorts are stable: sorting by x after (y, z) leaves (x, y, z, original index) order
        voxel_xkeys_kernel<<<blocks, kBlock, 0, st>>>(points, (int)n, v, w.idx_sorted, w.x_in);
        bytes = w.cub_bytes;
        if (cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, w.x_in, w.x_sorted, w.idx_sorted, w.idx_in, (int)n, 0, v.bits[0], st) != cudaSuccess)
            return pmb200_internal_launch_status("voxel_downsample (sort)");
        order = w.idx_in;
    }
    voxel_flags_kernel<<<blocks, kBlock, 0, st>>>(points, (int)n, v, order, w.flags);
    bytes = w.cub_bytes;
    if (cub::DeviceScan::InclusiveSum(w.cub_temp, bytes, w.flags, w.pos, (int)n, st) != cudaSuccess)
        return pmb200_internal_launch_status("voxel_downsample (scan)");
    voxel_runs_kernel<<<blocks, kBlock, 0, st>>>(w.flags, w.pos, (int)n, w.runs, reinterpret_cast<long long *>(count_out));
    voxel_mean_kernel<<<blocks, kBlock, 0, st>>>(points, order, w.runs, reinterpret_cast<const long long *>(count_out), points_out);
    return pmb200_internal_launch_status("voxel_downsample");
}

extern "C" int64_t pmb200_icp_target_workspace_bytes(int64_t n_target) {
    if (n_target < 0 || n_target >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "icp_target_workspace_bytes: 0 <= n_target < 2^31");
    Carver c{nullptr};
    Grid g;
    const long long b = icp_target_layout(c, n_target, g);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "icp_target_workspace_bytes: no CUDA device to size the CUB sort for") : b;
}

extern "C" int pmb200_icp_target(const double *target, int64_t n_target, double cell, void *target_workspace, int64_t workspace_bytes,
                                 void *stream) {
    if ((!target && n_target > 0) || !target_workspace) return pmb200_internal_fail(PMB200_EINVAL, "icp_target: null pointer");
    if (n_target < 0 || n_target >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "icp_target: 0 <= n_target < 2^31");
    if (!(cell > 0.0) || !(cell < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, "icp_target: cell must be positive and finite");
    Carver c{static_cast<char *>(target_workspace)};
    Grid g;
    const long long need = icp_target_layout(c, n_target, g);
    if (need < 0 || workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "icp_target: workspace smaller than icp_target_workspace_bytes(n_target)");
    if (n_target == 0) return 0;
    if (build_grid(g, target, (int)n_target, cell, true, reinterpret_cast<cudaStream_t>(stream)) != cudaSuccess)
        return pmb200_internal_launch_status("icp_target (sort)");
    return pmb200_internal_launch_status("icp_target");
}

extern "C" int64_t pmb200_icp_query_workspace_bytes(int64_t n_source) {
    if (n_source < 0 || n_source >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "icp_query_workspace_bytes: 0 <= n_source < 2^31");
    return (int64_t)align256((size_t)grid_blocks(n_source) * kMoments * sizeof(double));
}

extern "C" int pmb200_icp_query(const double *source, int64_t n_source, const double *transform_host, const double *origin_host,
                                double max_dist, const void *target_workspace, int64_t n_target, double cell, int *corr_out,
                                double *moments_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!source && n_source > 0) || !transform_host || !origin_host || !target_workspace || !moments_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "icp_query: null pointer");
    if (n_source < 0 || n_source >= (1ll << 31) || n_target < 0 || n_target >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "icp_query: 0 <= n_source, n_target < 2^31");
    if (!(max_dist > 0.0) || !(max_dist < INFINITY) || !(cell >= max_dist / kMaxCellsPerDist) || !(cell < INFINITY))
        return pmb200_internal_fail(PMB200_EINVAL, "icp_query: max_dist finite and positive, max_dist / 256 <= cell < inf");
    IcpParams p;
    if (!affine_from_host(transform_host, p.t))
        return pmb200_internal_fail(PMB200_EINVAL, "icp_query: the transform must be finite with last row 0 0 0 1");
    for (int a = 0; a < 3; ++a) {
        if (!(origin_host[a] > -INFINITY && origin_host[a] < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, "icp_query: origin must be finite");
        p.origin[a] = origin_host[a];
    }
    if (workspace_bytes < pmb200_icp_query_workspace_bytes(n_source))
        return pmb200_internal_fail(PMB200_EINVAL, "icp_query: workspace smaller than icp_query_workspace_bytes(n_source)");
    Carver c{const_cast<char *>(static_cast<const char *>(target_workspace))};
    Grid g;
    if (icp_target_layout(c, n_target, g) < 0) return pmb200_internal_fail(PMB200_EINVAL, "icp_query: no CUDA device to size the CUB sort for");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (n_source == 0 || n_target == 0) {  // no correspondences
        cudaMemsetAsync(moments_out, 0, kMoments * sizeof(double), st);
        if (n_source > 0 && corr_out) cudaMemsetAsync(corr_out, 0xff, (size_t)n_source * sizeof(int), st);
        return pmb200_internal_launch_status("icp_query");
    }
    p.src = source; p.n_src = (int)n_source; p.fine = g.fine; p.coarse = g.coarse; p.pts = g.pts; p.idx = g.idx_sorted;
    p.inv_cell = 1.0 / cell; p.cell = cell; p.max_dist = max_dist; p.corr = corr_out;
    p.partials = static_cast<double *>(workspace);
    const int blocks = grid_blocks(n_source);
    icp_query_kernel<<<blocks, kBlock, 0, st>>>(p);
    icp_finish_kernel<<<1, kBlock, 0, st>>>(p.partials, blocks, moments_out);
    return pmb200_internal_launch_status("icp_query");
}
