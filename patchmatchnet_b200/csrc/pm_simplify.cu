// pm_simplify.cu -- quadric edge-collapse simplification of triangle meshes in rounds of independent collapses (beyond the
// reference; definition in include/patchmatch_b200.h, INTEGRATION.md "Mesh simplification (beyond the reference)").
//
// Per round, from the current face list: three edge keys per face, CUB radix sort and run-length encoding into the edges
// with their face counts; a vertex -> face CSR from sorted (vertex, face) keys; one thread per edge for validity, placement
// and cost (pm_simplify_math.cuh); 64-bit atomicMin of the keys per vertex, then per neighbourhood; selection; the
// collapses; a stable compaction of the faces.  The only floating-point work is per thread, in a fixed order: no atomics
// touch a float, so reruns give the same bits.  One host read per round (the selected count and the faces it removes).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_simplify_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmsimp;

constexpr int kBlock = 256;
constexpr long long kMaxVertices = (1ll << 31) - 1;  // nv + 1 offsets stay int (CUB item counts)
constexpr long long kMaxFaces = 1ll << 29;  // 3 edge keys per face stay below 2^31 (CUB item counts are int)
constexpr unsigned long long kNone = ~0ull;

struct Face {
    int v[3];
};

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct Carver {  // bump allocator over the caller's workspace; a NULL base only measures
    char *base;
    size_t used = 0;
    template <typename T>
    T *take(size_t count) {
        T *p = base ? reinterpret_cast<T *>(base + used) : nullptr;
        used += align256((count < 1 ? 1 : count) * sizeof(T));
        return p;
    }
};

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 ? 65535 : b));
}

inline int bits_for(long long n) {  // bits that hold 0..n-1, at least 1
    int b = 1;
    while ((1ll << b) < n) ++b;
    return b;
}

// counters on the device: [0] edges, [1] selected, [2] faces the selected remove, [3] kept after the target, [4] faces the
// kept remove, [5] component labels changed, [6] surviving vertices, [7] faces after a compaction
struct Layout {
    double *pos, *q;
    unsigned char *col, *bnd, *lck, *fflag;
    int *rep, *lab, *deg, *off;
    unsigned long long *mkey, *Mkey;
    Face *fa, *fb;
    unsigned long long *ek_in, *ek, *vf_in, *vf, *edges, *cand;
    int *ecount;
    int *sel, *sel_sorted, *rem, *rem_scan;
    unsigned long long *selkey, *selkey_sorted;
    long long *ctr;
    void *cub;
    size_t cub_bytes;
};

bool layout(Carver &c, long long nv, long long nf, Layout &l) {
    const long long ne = 3 * nf;
    l.pos = c.take<double>(3 * nv);
    l.q = c.take<double>(kQ * nv);
    l.col = c.take<unsigned char>(3 * nv);
    l.bnd = c.take<unsigned char>(nv);
    l.lck = c.take<unsigned char>(nv);
    l.rep = c.take<int>(nv);
    l.lab = c.take<int>(nv + 1);
    l.deg = c.take<int>(nv + 1);
    l.off = c.take<int>(nv + 1);
    l.mkey = c.take<unsigned long long>(nv);
    l.Mkey = c.take<unsigned long long>(nv);
    l.fa = c.take<Face>(nf);
    l.fb = c.take<Face>(nf);
    l.fflag = c.take<unsigned char>(nf);
    l.ek_in = c.take<unsigned long long>(ne);
    l.ek = c.take<unsigned long long>(ne);
    l.vf_in = c.take<unsigned long long>(ne);
    l.vf = c.take<unsigned long long>(ne);
    l.edges = c.take<unsigned long long>(ne);
    l.cand = c.take<unsigned long long>(ne);
    l.ecount = c.take<int>(ne);
    const long long ns = nv / 2 + 1;  // selected edges share no endpoint
    l.sel = c.take<int>(ns);
    l.sel_sorted = c.take<int>(ns);
    l.rem = c.take<int>(ns);
    l.rem_scan = c.take<int>(ns);
    l.selkey = c.take<unsigned long long>(ns);
    l.selkey_sorted = c.take<unsigned long long>(ns);
    l.ctr = c.take<long long>(8);
    size_t m = 0, b = 0;
    const int ine = (int)(ne < 1 ? 1 : ne), inv = (int)(nv + 1), ins = (int)ns, inf = (int)(nf < 1 ? 1 : nf);
    using U = unsigned long long;
    if (cub::DeviceRadixSort::SortKeys(nullptr, b, (U *)nullptr, (U *)nullptr, ine) != cudaSuccess) return false;
    m = b > m ? b : m;
    if (cub::DeviceRunLengthEncode::Encode(nullptr, b, (U *)nullptr, (U *)nullptr, (int *)nullptr, (long long *)nullptr, ine) != cudaSuccess)
        return false;
    m = b > m ? b : m;
    if (cub::DeviceScan::ExclusiveSum(nullptr, b, (int *)nullptr, (int *)nullptr, inv) != cudaSuccess) return false;
    m = b > m ? b : m;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b, (U *)nullptr, (U *)nullptr, (int *)nullptr, (int *)nullptr, ins) != cudaSuccess) return false;
    m = b > m ? b : m;
    if (cub::DeviceScan::InclusiveSum(nullptr, b, (int *)nullptr, (int *)nullptr, ins) != cudaSuccess) return false;
    m = b > m ? b : m;
    if (cub::DeviceSelect::Flagged(nullptr, b, (Face *)nullptr, (unsigned char *)nullptr, (Face *)nullptr, (long long *)nullptr, inf) !=
        cudaSuccess)
        return false;
    m = b > m ? b : m;
    l.cub_bytes = m;
    l.cub = c.take<char>(m);
    return true;
}

#define GRID_LOOP(i, n) for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < (n); i += (long long)gridDim.x * kBlock)

__global__ void __launch_bounds__(kBlock) init_vertices_kernel(const float *xyz, const unsigned char *rgb, int nv, double *pos,
                                                               unsigned char *col, int *rep, int *lab) {
    GRID_LOOP(v, nv) {
        for (int c = 0; c < 3; ++c) {
            pos[3 * v + c] = (double)xyz[3 * v + c];
            col[3 * v + c] = rgb ? rgb[3 * v + c] : 0;
        }
        rep[v] = (int)v;
        lab[v] = (int)v;
    }
}

// a face is kept when its indices are in range and distinct
__global__ void __launch_bounds__(kBlock) input_flags_kernel(const int *faces, long long nf, int nv, unsigned char *flag) {
    GRID_LOOP(f, nf) {
        const int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
        flag[f] = (a >= 0 && a < nv && b >= 0 && b < nv && c >= 0 && c < nv && a != b && b != c && a != c) ? 1 : 0;
    }
}

// ---- components: min-label propagation with hooking and pointer jumping; the fixed point is each component's smallest vertex

__global__ void __launch_bounds__(kBlock) hook_kernel(const Face *f, long long nf, int *lab, long long *changed) {
    GRID_LOOP(i, nf) {
        const Face t = f[i];
        int m = lab[t.v[0]];
        m = min(m, lab[t.v[1]]);
        m = min(m, lab[t.v[2]]);
        for (int k = 0; k < 3; ++k) {
            const int old = atomicMin(&lab[t.v[k]], m);
            if (old > m) {
                atomicMin(&lab[old], m);
                *changed = 1;
            }
        }
    }
}

__global__ void __launch_bounds__(kBlock) jump_kernel(int *lab, int nv) {
    GRID_LOOP(v, nv) {
        const int l = lab[v];
        const int ll = lab[l];
        if (ll < l) atomicMin(&lab[v], ll);
    }
}

__global__ void __launch_bounds__(kBlock) component_count_kernel(const Face *f, long long nf, const int *lab, int *count) {
    GRID_LOOP(i, nf) atomicAdd(&count[lab[f[i].v[0]]], 1);
}

__global__ void __launch_bounds__(kBlock) component_flags_kernel(const Face *f, long long nf, const int *lab, const int *count, long long F,
                                                                 unsigned char *flag) {
    GRID_LOOP(i, nf) flag[i] = count[lab[f[i].v[0]]] >= F ? 1 : 0;
}

// ---- topology of a round ----------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) face_keys_kernel(const Face *f, long long nf, int vb, int fbits, unsigned long long *ek,
                                                           unsigned long long *vf, int *deg) {
    GRID_LOOP(i, nf) {
        const Face t = f[i];
        for (int k = 0; k < 3; ++k) {
            const unsigned long long a = (unsigned long long)t.v[k], b = (unsigned long long)t.v[k == 2 ? 0 : k + 1];
            ek[3 * i + k] = a < b ? (a << vb) | b : (b << vb) | a;
            vf[3 * i + k] = (a << fbits) | (unsigned long long)i;
            atomicAdd(&deg[t.v[k]], 1);
        }
    }
}

__global__ void __launch_bounds__(kBlock) edge_flags_kernel(const unsigned long long *edges, const int *ecount, const long long *n_edges,
                                                            int vb, unsigned char *bnd, unsigned char *lck) {
    const unsigned long long mask = (1ull << vb) - 1;
    GRID_LOOP(e, *n_edges) {
        const int a = (int)(edges[e] >> vb), b = (int)(edges[e] & mask), c = ecount[e];
        if (c == 1) bnd[a] = bnd[b] = 1;
        if (c > 2) lck[a] = lck[b] = 1;
    }
}

// vertex-indexed arrays are addressed in 64 bits: 10 * v overflows int from v = 214,748,365
__device__ __forceinline__ const double *P(const double *pos, long long v) { return pos + 3 * v; }

__device__ __forceinline__ int edge_count(const unsigned long long *edges, const int *ecount, long long n, unsigned long long key) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (edges[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && edges[lo] == key) ? ecount[lo] : 0;
}

// Quadrics, once: incident faces by ascending index, then border edges by ascending key
__global__ void __launch_bounds__(kBlock) quadric_kernel(const Face *f, const unsigned long long *vf, const int *off, const double *pos,
                                                         const unsigned long long *edges, const int *ecount, const long long *n_edges,
                                                         int nv, int vb, int fbits, double *qout) {
    const unsigned long long fmask = (1ull << fbits) - 1;
    const long long ne = *n_edges;
    GRID_LOOP(v, nv) {
        double q[kQ];
        for (int k = 0; k < kQ; ++k) q[k] = 0.0;
        const int s0 = off[v], s1 = off[v + 1];
        for (int s = s0; s < s1; ++s) {
            const Face t = f[vf[s] & fmask];
            add_face_quadric(P(pos, t.v[0]), P(pos, t.v[1]), P(pos, t.v[2]), q);
        }
        unsigned long long last = 0;
        bool first = true;
        for (;;) {
            unsigned long long best = kNone;
            int bf = -1;
            for (int s = s0; s < s1; ++s) {
                const int fi = (int)(vf[s] & fmask);
                const Face t = f[fi];
                for (int k = 0; k < 3; ++k) {
                    const unsigned long long w = (unsigned long long)t.v[k];
                    if ((long long)w == v) continue;
                    const unsigned long long vv = (unsigned long long)v;
                    const unsigned long long key = vv < w ? (vv << vb) | w : (w << vb) | vv;
                    if ((!first && key <= last) || key >= best) continue;
                    if (edge_count(edges, ecount, ne, key) == 1) {
                        best = key;
                        bf = fi;
                    }
                }
            }
            if (bf < 0) break;
            const Face t = f[bf];
            const int a = (int)(best >> vb), b = (int)(best & ((1ull << vb) - 1));
            add_border_quadric(P(pos, a), P(pos, b), P(pos, t.v[0]), P(pos, t.v[1]), P(pos, t.v[2]), q);
            last = best;
            first = false;
        }
        for (int k = 0; k < kQ; ++k) qout[kQ * v + k] = q[k];
    }
}

__device__ __forceinline__ bool has(const Face &t, int x) { return t.v[0] == x || t.v[1] == x || t.v[2] == x; }

// the two vertices of t other than a
__device__ __forceinline__ void others(const Face &t, int a, int &x, int &y) {
    const int k = t.v[0] == a ? 0 : (t.v[1] == a ? 1 : 2);
    x = t.v[k == 2 ? 0 : k + 1];
    y = t.v[k == 0 ? 2 : k - 1];
}

__device__ __forceinline__ int slot_of(const Face &t, int a) { return t.v[0] == a ? 0 : (t.v[1] == a ? 1 : 2); }

__device__ __forceinline__ void qsum(const double *q, long long a, long long b, double *o) {
    for (int k = 0; k < kQ; ++k) o[k] = add64(q[kQ * a + k], q[kQ * b + k]);
}

// no face of c's star without o flips or becomes zero-area when c moves to v
__device__ __forceinline__ bool star_keeps(const Face *f, const unsigned long long *vf, unsigned long long fmask, const double *pos, int s0,
                                           int s1, int c, int o, const double *v) {
    for (int s = s0; s < s1; ++s) {
        const Face t = f[vf[s] & fmask];
        if (has(t, o)) continue;
        if (!face_keeps_orientation(P(pos, t.v[0]), P(pos, t.v[1]), P(pos, t.v[2]), slot_of(t, c), v)) return false;
    }
    return true;
}

// Candidate (a, b): validity, placement, cost -> key (kNone when invalid); atomicMin into m of both endpoints
__global__ void __launch_bounds__(kBlock) evaluate_kernel(const Face *f, const unsigned long long *vf, const int *off, const double *pos,
                                                          const double *qv, const unsigned char *bnd, const unsigned char *lck,
                                                          const unsigned long long *edges, const int *ecount, const long long *n_edges,
                                                          int vb, int fbits, unsigned long long *cand, unsigned long long *mkey) {
    const unsigned long long fmask = (1ull << fbits) - 1, vmask = (1ull << vb) - 1;
    GRID_LOOP(e, *n_edges) {
        const int a = (int)(edges[e] >> vb), b = (int)(edges[e] & vmask), cnt = ecount[e];
        const int a0 = off[a], a1 = off[a + 1], b0 = off[b], b1 = off[b + 1];
        bool ok = cnt <= 2 && !lck[a] && !lck[b] && a1 - a0 <= kMaxValence && b1 - b0 <= kMaxValence && !(cnt == 2 && bnd[a] && bnd[b]);
        int opp0 = -1, opp1 = -1;  // the opposite vertices (cnt <= 2)
        if (ok)
            for (int s = a0; s < a1; ++s) {
                const Face t = f[vf[s] & fmask];
                if (!has(t, b)) continue;
                int x, y;
                others(t, a, x, y);
                const int o = x == b ? y : x;
                if (opp0 < 0) opp0 = o;
                else opp1 = o;
            }
        // link condition: every common neighbour is opposite, and no (x, y) spans both a-x-y and b-x-y
        for (int s = a0; ok && s < a1; ++s) {
            const Face t = f[vf[s] & fmask];
            if (has(t, b)) continue;
            int x, y;
            others(t, a, x, y);
            bool hx = false, hy = false, hxy = false;
            for (int r = b0; r < b1; ++r) {
                const Face u = f[vf[r] & fmask];
                const bool ux = has(u, x), uy = has(u, y);
                hx |= ux;
                hy |= uy;
                hxy |= ux && uy;
            }
            if (hxy || (hx && x != opp0 && x != opp1) || (hy && y != opp0 && y != opp1)) ok = false;
        }
        unsigned long long key = kNone;
        if (ok) {
            double q[kQ], v[3];
            qsum(qv, a, b, q);
            placement(q, P(pos, a), P(pos, b), v);
            ok = star_keeps(f, vf, fmask, pos, a0, a1, a, b, v) && star_keeps(f, vf, fmask, pos, b0, b1, b, a, v);
            if (ok) key = edge_key(quadric_cost(q, v), (unsigned int)e);
        }
        cand[e] = key;
        if (key != kNone) {
            atomicMin(&mkey[a], key);
            atomicMin(&mkey[b], key);
        }
    }
}

// M(v) = min of m over v and its neighbours (Mkey starts as a copy of mkey)
__global__ void __launch_bounds__(kBlock) neighbour_min_kernel(const unsigned long long *edges, const long long *n_edges, int vb,
                                                               const unsigned long long *mkey, unsigned long long *Mkey) {
    const unsigned long long vmask = (1ull << vb) - 1;
    GRID_LOOP(e, *n_edges) {
        const int a = (int)(edges[e] >> vb), b = (int)(edges[e] & vmask);
        if (mkey[b] != kNone) atomicMin(&Mkey[a], mkey[b]);
        if (mkey[a] != kNone) atomicMin(&Mkey[b], mkey[a]);
    }
}

__global__ void __launch_bounds__(kBlock) select_kernel(const unsigned long long *edges, const int *ecount, const unsigned long long *cand,
                                                        const long long *n_edges, int vb, const unsigned long long *Mkey, int *sel,
                                                        unsigned long long *selkey, int *rem, long long *ctr) {
    const unsigned long long vmask = (1ull << vb) - 1;
    GRID_LOOP(e, *n_edges) {
        const unsigned long long k = cand[e];
        if (k == kNone) continue;
        const int a = (int)(edges[e] >> vb), b = (int)(edges[e] & vmask);
        if (k != Mkey[a] || k != Mkey[b]) continue;
        const int i = (int)atomicAdd((unsigned long long *)&ctr[1], 1ull);
        sel[i] = (int)e;
        selkey[i] = k;
        rem[i] = ecount[e];
        atomicAdd((unsigned long long *)&ctr[2], (unsigned long long)ecount[e]);
    }
}

// the kept prefix in key order: edge i is kept when the faces the edges before it remove are fewer than `need`
__global__ void __launch_bounds__(kBlock) kept_count_kernel(const int *scan, const int *rem, long long ns, long long need, long long *ctr) {
    GRID_LOOP(i, ns) {
        const long long incl = scan[i], excl = incl - rem[i];
        if (excl < need && incl >= need) {
            ctr[3] = i + 1;
            ctr[4] = incl;
        }
    }
}

__global__ void __launch_bounds__(kBlock) apply_kernel(const int *sel, const long long *n_kept, const unsigned long long *edges, int vb,
                                                       double *pos, double *qv, unsigned char *col, int *rep) {
    const unsigned long long vmask = (1ull << vb) - 1;
    GRID_LOOP(i, *n_kept) {
        const int e = sel[i];
        const long long a = (long long)(edges[e] >> vb), b = (long long)(edges[e] & vmask);
        double q[kQ], v[3];
        qsum(qv, a, b, q);
        placement(q, P(pos, a), P(pos, b), v);
        unsigned char c[3];
        placement_colour(P(pos, a), P(pos, b), v, col + 3 * a, col + 3 * b, c);
        for (int k = 0; k < 3; ++k) {
            pos[3 * a + k] = v[k];
            col[3 * a + k] = c[k];
        }
        for (int k = 0; k < kQ; ++k) qv[kQ * a + k] = q[k];
        rep[b] = (int)a;
    }
}

__global__ void __launch_bounds__(kBlock) remap_faces_kernel(Face *f, long long nf, const int *rep, unsigned char *flag) {
    GRID_LOOP(i, nf) {
        Face t = f[i];
        for (int k = 0; k < 3; ++k) t.v[k] = rep[t.v[k]];
        f[i] = t;
        flag[i] = (t.v[0] != t.v[1] && t.v[1] != t.v[2] && t.v[0] != t.v[2]) ? 1 : 0;
    }
}

__global__ void __launch_bounds__(kBlock) mark_used_kernel(const Face *f, long long nf, int *used) {
    GRID_LOOP(i, nf) for (int k = 0; k < 3; ++k) used[f[i].v[k]] = 1;
}

__global__ void __launch_bounds__(kBlock) write_vertices_kernel(const double *pos, const unsigned char *col, const int *used,
                                                                const int *idx, int nv, float *xyz, unsigned char *rgb) {
    GRID_LOOP(v, nv) {
        if (!used[v]) continue;
        const long long o = idx[v];
        for (int c = 0; c < 3; ++c) {
            xyz[3 * o + c] = (float)pos[3 * v + c];
            if (rgb) rgb[3 * o + c] = col[3 * v + c];
        }
    }
}

__global__ void __launch_bounds__(kBlock) write_faces_kernel(const Face *f, long long nf, const int *idx, int *out) {
    GRID_LOOP(i, nf) for (int k = 0; k < 3; ++k) out[3 * i + k] = idx[f[i].v[k]];
}

int check_sizes(const char *what, int64_t nv, int64_t nf) {
    if (nv < 0 || nv >= kMaxVertices || nf < 0 || nf >= kMaxFaces) {
        char msg[160];
        snprintf(msg, sizeof msg, "%s: 0 <= n_vertices < 2^31 - 1 and 0 <= n_faces < 2^29", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    return 0;
}

int read_counters(long long *host, const long long *dev, int n, cudaStream_t st, const char *what) {
    if (cudaMemcpyAsync(host, dev, n * sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status(what);
    return 0;
}

// stable compaction of faces by flag: src -> dst, the count to ctr[7]
int compact(const Layout &l, const Face *src, Face *dst, long long nf, cudaStream_t st) {
    size_t bytes = l.cub_bytes;
    if (cub::DeviceSelect::Flagged(l.cub, bytes, src, l.fflag, dst, l.ctr + 7, (int)nf, st) != cudaSuccess)
        return pmb200_internal_launch_status("simplify_mesh (compact)");
    return 0;
}

}  // namespace

extern "C" int64_t pmb200_simplify_mesh_workspace_bytes(int64_t n_vertices, int64_t n_faces) {
    if (const int rc = check_sizes("simplify_mesh_workspace_bytes", n_vertices, n_faces)) return rc;
    Carver c{nullptr};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l))
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh_workspace_bytes: no CUDA device to size the CUB passes for");
    return (int64_t)c.used;
}

extern "C" int pmb200_simplify_mesh(const float *xyz, const unsigned char *rgb, int64_t n_vertices, const int *faces, int64_t n_faces,
                                    int64_t target_faces, int64_t min_component_faces, int64_t *counts_host, void *workspace,
                                    int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !counts_host || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh: null pointer");
    if (const int rc = check_sizes("simplify_mesh", n_vertices, n_faces)) return rc;
    if (target_faces < 0 || min_component_faces < 0)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh: target_faces and min_component_faces must be >= 0");
    Carver c{static_cast<char *>(workspace)};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh: workspace smaller than simplify_mesh_workspace_bytes(nv, nf)");
    counts_host[0] = counts_host[1] = counts_host[2] = 0;
    if (n_vertices == 0 || n_faces == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int nv = (int)n_vertices;
    const int vb = bits_for(nv), fbits = bits_for(n_faces);
    long long host[8];
    int rc;
    cudaMemsetAsync(l.ctr, 0, 8 * sizeof(long long), st);
    init_vertices_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(xyz, rgb, nv, l.pos, l.col, l.rep, l.lab);
    input_flags_kernel<<<grid_blocks(n_faces), kBlock, 0, st>>>(faces, n_faces, nv, l.fflag);
    if ((rc = compact(l, reinterpret_cast<const Face *>(faces), l.fa, n_faces, st))) return rc;
    if ((rc = read_counters(host, l.ctr, 8, st, "simplify_mesh"))) return rc;
    long long nf = host[7];
    if (min_component_faces > 0 && nf > 0) {
        for (;;) {
            cudaMemsetAsync(l.ctr + 5, 0, sizeof(long long), st);
            hook_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, l.lab, l.ctr + 5);
            jump_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(l.lab, nv);
            if ((rc = read_counters(host + 5, l.ctr + 5, 1, st, "simplify_mesh (components)"))) return rc;
            if (!host[5]) break;
        }
        cudaMemsetAsync(l.deg, 0, (nv + 1) * sizeof(int), st);
        component_count_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, l.lab, l.deg);
        component_flags_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, l.lab, l.deg, min_component_faces, l.fflag);
        if ((rc = compact(l, l.fa, l.fb, nf, st))) return rc;
        if ((rc = read_counters(host + 7, l.ctr + 7, 1, st, "simplify_mesh (components)"))) return rc;
        nf = host[7];
        cudaMemcpyAsync(l.fa, l.fb, nf * sizeof(Face), cudaMemcpyDeviceToDevice, st);
    }
    long long rounds = 0;
    size_t bytes;
    while (nf > target_faces) {
        const long long ne = 3 * nf;
        cudaMemsetAsync(l.deg, 0, (nv + 1) * sizeof(int), st);
        cudaMemsetAsync(l.ctr, 0, 5 * sizeof(long long), st);
        face_keys_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, vb, fbits, l.ek_in, l.vf_in, l.deg);
        bytes = l.cub_bytes;
        if (cub::DeviceRadixSort::SortKeys(l.cub, bytes, l.ek_in, l.ek, (int)ne, 0, 2 * vb, st) != cudaSuccess)
            return pmb200_internal_launch_status("simplify_mesh (edge sort)");
        bytes = l.cub_bytes;
        if (cub::DeviceRunLengthEncode::Encode(l.cub, bytes, l.ek, l.edges, l.ecount, l.ctr, (int)ne, st) != cudaSuccess)
            return pmb200_internal_launch_status("simplify_mesh (edges)");
        bytes = l.cub_bytes;
        if (cub::DeviceRadixSort::SortKeys(l.cub, bytes, l.vf_in, l.vf, (int)ne, 0, vb + fbits, st) != cudaSuccess)
            return pmb200_internal_launch_status("simplify_mesh (vertex-face sort)");
        bytes = l.cub_bytes;
        if (cub::DeviceScan::ExclusiveSum(l.cub, bytes, l.deg, l.off, nv + 1, st) != cudaSuccess)
            return pmb200_internal_launch_status("simplify_mesh (offsets)");
        cudaMemsetAsync(l.bnd, 0, nv, st);
        cudaMemsetAsync(l.lck, 0, nv, st);
        edge_flags_kernel<<<grid_blocks(ne), kBlock, 0, st>>>(l.edges, l.ecount, l.ctr, vb, l.bnd, l.lck);
        if (rounds == 0)
            quadric_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(l.fa, l.vf, l.off, l.pos, l.edges, l.ecount, l.ctr, nv, vb, fbits, l.q);
        cudaMemsetAsync(l.mkey, 0xff, nv * sizeof(unsigned long long), st);
        evaluate_kernel<<<grid_blocks(ne), kBlock, 0, st>>>(l.fa, l.vf, l.off, l.pos, l.q, l.bnd, l.lck, l.edges, l.ecount, l.ctr, vb, fbits,
                                                             l.cand, l.mkey);
        cudaMemcpyAsync(l.Mkey, l.mkey, nv * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st);
        neighbour_min_kernel<<<grid_blocks(ne), kBlock, 0, st>>>(l.edges, l.ctr, vb, l.mkey, l.Mkey);
        select_kernel<<<grid_blocks(ne), kBlock, 0, st>>>(l.edges, l.ecount, l.cand, l.ctr, vb, l.Mkey, l.sel, l.selkey, l.rem, l.ctr);
        if ((rc = read_counters(host, l.ctr, 3, st, "simplify_mesh (select)"))) return rc;
        const long long ns = host[1];
        if (ns == 0) break;
        long long removed = host[2];
        const int *kept = l.sel;
        if (nf - removed < target_faces) {  // the target bites: the shortest prefix in key order
            bytes = l.cub_bytes;
            if (cub::DeviceRadixSort::SortPairs(l.cub, bytes, l.selkey, l.selkey_sorted, l.sel, l.sel_sorted, (int)ns, 0, 64, st) != cudaSuccess)
                return pmb200_internal_launch_status("simplify_mesh (target sort)");
            // the removal counts in key order: gather through the sorted edge indices
            bytes = l.cub_bytes;
            if (cub::DeviceRadixSort::SortPairs(l.cub, bytes, l.selkey, l.selkey_sorted, l.rem, l.rem_scan, (int)ns, 0, 64, st) != cudaSuccess)
                return pmb200_internal_launch_status("simplify_mesh (target sort)");
            bytes = l.cub_bytes;
            cudaMemcpyAsync(l.rem, l.rem_scan, ns * sizeof(int), cudaMemcpyDeviceToDevice, st);
            if (cub::DeviceScan::InclusiveSum(l.cub, bytes, l.rem, l.rem_scan, (int)ns, st) != cudaSuccess)
                return pmb200_internal_launch_status("simplify_mesh (target scan)");
            kept_count_kernel<<<grid_blocks(ns), kBlock, 0, st>>>(l.rem_scan, l.rem, ns, nf - target_faces, l.ctr);
            if ((rc = read_counters(host, l.ctr, 5, st, "simplify_mesh (target)"))) return rc;
            removed = host[4];
            kept = l.sel_sorted;
        } else {
            cudaMemcpyAsync(l.ctr + 3, l.ctr + 1, sizeof(long long), cudaMemcpyDeviceToDevice, st);
        }
        apply_kernel<<<grid_blocks(ns), kBlock, 0, st>>>(kept, l.ctr + 3, l.edges, vb, l.pos, l.q, l.col, l.rep);
        remap_faces_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, l.rep, l.fflag);
        if ((rc = compact(l, l.fa, l.fb, nf, st))) return rc;
        Face *t = l.fa;
        l.fa = l.fb;
        l.fb = t;
        nf -= removed;
        ++rounds;
    }
    if (rounds % 2) {  // the result goes where the write call looks: the first face buffer
        cudaMemcpyAsync(l.fb, l.fa, nf * sizeof(Face), cudaMemcpyDeviceToDevice, st);
        Face *t = l.fa;
        l.fa = l.fb;
        l.fb = t;
    }
    // surviving vertices: referenced by a face, numbered in ascending original index
    cudaMemsetAsync(l.deg, 0, (nv + 1) * sizeof(int), st);
    mark_used_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(l.fa, nf, l.deg);
    bytes = l.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(l.cub, bytes, l.deg, l.lab, nv + 1, st) != cudaSuccess)
        return pmb200_internal_launch_status("simplify_mesh (vertex numbering)");
    long long nv_out = 0;
    int tail = 0;
    if (cudaMemcpyAsync(&tail, l.lab + nv, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status("simplify_mesh");
    nv_out = tail;
    counts_host[0] = nv_out;
    counts_host[1] = nf;
    counts_host[2] = rounds;
    return pmb200_internal_launch_status("simplify_mesh");
}

extern "C" int pmb200_simplify_mesh_write(int64_t n_vertices, int64_t n_faces, int64_t n_faces_out, float *xyz_out,
                                          unsigned char *rgb_out, int *faces_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if (((!xyz_out || !faces_out) && n_faces_out > 0) || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh_write: null pointer");
    if (const int rc = check_sizes("simplify_mesh_write", n_vertices, n_faces)) return rc;
    if (n_faces_out < 0 || n_faces_out > n_faces)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh_write: 0 <= n_faces_out <= n_faces");
    Carver c{static_cast<char *>(workspace)};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "simplify_mesh_write: workspace smaller than simplify_mesh_workspace_bytes(nv, nf)");
    if (n_vertices == 0 || n_faces_out == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    write_vertices_kernel<<<grid_blocks(n_vertices), kBlock, 0, st>>>(l.pos, l.col, l.deg, l.lab, (int)n_vertices, xyz_out, rgb_out);
    write_faces_kernel<<<grid_blocks(n_faces_out), kBlock, 0, st>>>(l.fa, n_faces_out, l.lab, faces_out);
    return pmb200_internal_launch_status("simplify_mesh_write");
}
