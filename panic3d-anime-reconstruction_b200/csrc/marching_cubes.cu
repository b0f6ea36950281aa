// Marching cubes on the device (p3d_mesh.h): the mesh of the eval's density volume without a host round trip
// (reference _util/eg3d_metrics3d.py:186-211, skimage Lewiner on the CPU).  Rules: DESIGN.md section 2, "Marching cubes".
//
//   k_mc_count   thread per node: its sign-change edges along +a, +b, +c (0-3 vertices) and, when it is the lower corner
//                of a cell, that cell's non-degenerate triangles; both counts packed in one u64 (vertices low word,
//                triangles high word) -> one in-place CUB exclusive scan gives every node its vertex and triangle offsets
//   k_mc_emit    the same walk again, writing the vertices at their scanned offsets and the triangles, whose indices are
//                the owner node's offset plus the popcount of its lower-axis edge bits
//
// Memory-bound stencil work: consecutive threads own consecutive nodes along c, so each of the 8 corner loads of a cell is
// a coalesced row read and the 8-fold corner reuse between neighbouring cells is served by L1.  Empty cells (case 0 or
// 255) exit after the corner loads.  The triangulation is built per cell at run time (no table): the segments of the six
// faces (asymptotic decider on ambiguous faces) are chained into loops, each fanned from its smallest vertex.
#include <cub/device/device_scan.cuh>

#include "render_device.cuh"
#include "../../include/p3d_mesh.h"

namespace p3d {

namespace {

constexpr int kThreads = 256;
constexpr size_t kHead = 256;                    // workspace head: the exact totals (2 x u64, atomics)
constexpr long long kMaxNodes = 1ll << 30;       // keeps the packed vertex prefix below 2^32 (3 vertices per node at most)

// corner k of a cell: offset ((k >> 2) & 1, (k >> 1) & 1, k & 1) along axes (0, 1, 2)
// local edge e = (lower corner, axis), sorted by corner then axis: the order of the global vertex indices they own
__constant__ unsigned char kEdgeCorner[12] = {0, 0, 0, 1, 1, 2, 2, 3, 4, 4, 5, 6};
__constant__ unsigned char kEdgeAxis[12] = {0, 1, 2, 0, 1, 0, 2, 0, 1, 2, 1, 2};
// faces: corners in counter-clockwise order seen from outside the cell, the local edges between consecutive corners
// (kFaceEdge[f][k] joins kFaceCyc[f][k] and kFaceCyc[f][k+1]), and the corners at (u,w) = (0,0), (0,1), (1,0), (1,1)
// with u < w the face's in-plane axes - the order the asymptotic decider reads them in, the same from both cells
__constant__ unsigned char kFaceCyc[6][4] = {{0, 1, 3, 2}, {4, 6, 7, 5}, {0, 4, 5, 1}, {2, 3, 7, 6}, {0, 2, 6, 4}, {1, 5, 7, 3}};
__constant__ unsigned char kFaceEdge[6][4] = {{2, 4, 6, 1}, {8, 11, 10, 9}, {0, 9, 3, 2}, {6, 7, 11, 5}, {1, 5, 8, 0}, {3, 10, 7, 4}};
__constant__ unsigned char kFaceCanon[6][4] = {{0, 1, 2, 3}, {4, 5, 6, 7}, {0, 1, 4, 5}, {2, 3, 6, 7}, {0, 2, 4, 6}, {1, 3, 5, 7}};

struct Node {
    long long n;           // flat index
    int a, b, c;
};

__device__ __forceinline__ Node node_of(long long n, int d1, int d2) {
    Node r;
    r.n = n;
    r.c = (int)(n % d2);
    const long long q = n / d2;
    r.b = (int)(q % d1);
    r.a = (int)(q / d1);
    return r;
}

struct Cell {
    float cv[8];           // corner values
    float t[12];           // edge parameter of every sign-change edge
    unsigned em;           // sign-change edges (bit e)
    unsigned char nxt[12]; // loop successor of each sign-change edge
};

// one segment per face crossing: from the edge the counter-clockwise walk enters the inside region through to the edge it
// leaves it by; on an ambiguous face the decider's saddle value picks which pair of corners the segments cut off
__device__ __forceinline__ void cell_build(Cell& c, unsigned ins, float level) {
    c.em = 0;
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        const int k = kEdgeCorner[e], k2 = k | (4 >> kEdgeAxis[e]);
        if (((ins >> k) ^ (ins >> k2)) & 1u) {
            c.em |= 1u << e;
            c.t[e] = __fdiv_rn(__fsub_rn(level, c.cv[k]), __fsub_rn(c.cv[k2], c.cv[k]));
        }
    }
#pragma unroll
    for (int f = 0; f < 6; ++f) {
        int in[4], fe[4], n_in = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            in[k] = (ins >> kFaceCyc[f][k]) & 1u;
            fe[k] = kFaceEdge[f][k];
            n_in += in[k];
        }
        if (n_in == 0 || n_in == 4) continue;
        if (n_in == 2 && in[0] == in[2]) {
            const float v00 = c.cv[kFaceCanon[f][0]], v01 = c.cv[kFaceCanon[f][1]];
            const float v10 = c.cv[kFaceCanon[f][2]], v11 = c.cv[kFaceCanon[f][3]];
            const float s = __fdiv_rn(__fsub_rn(__fmul_rn(v00, v11), __fmul_rn(v01, v10)),
                                      __fsub_rn(__fsub_rn(__fadd_rn(v00, v11), v01), v10));
            const bool connected = s > level;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (in[k] && !connected) c.nxt[fe[(k + 3) & 3]] = (unsigned char)fe[k];       // cut off the inside corner
                else if (!in[k] && connected) c.nxt[fe[k]] = (unsigned char)fe[(k + 3) & 3];  // cut off the outside corner
            }
        } else {
            int st = 0, en = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (!in[k] && in[(k + 1) & 3]) st = fe[k];
                if (in[k] && !in[(k + 1) & 3]) en = fe[k];
            }
            c.nxt[st] = (unsigned char)en;
        }
    }
}

// index-space position of the vertex on local edge e of the cell whose lower corner is (a, b, c)
__device__ __forceinline__ void edge_pos(const Cell& c, int e, int a, int b, int cc, float& x, float& y, float& z) {
    const int k = kEdgeCorner[e], ax = kEdgeAxis[e];
    x = (float)(a + ((k >> 2) & 1));
    y = (float)(b + ((k >> 1) & 1));
    z = (float)(cc + (k & 1));
    if (ax == 0) x = __fadd_rn(x, c.t[e]);
    else if (ax == 1) y = __fadd_rn(y, c.t[e]);
    else z = __fadd_rn(z, c.t[e]);
}

__device__ __forceinline__ bool same_pos(const Cell& c, int e0, int e1, const Node& nd) {
    float x0, y0, z0, x1, y1, z1;
    edge_pos(c, e0, nd.a, nd.b, nd.c, x0, y0, z0);
    edge_pos(c, e1, nd.a, nd.b, nd.c, x1, y1, z1);
    return x0 == x1 && y0 == y1 && z0 == z1;
}

// loops in order of their smallest edge, each fanned from it: tri(e_root, e_i, e_i+1) for the non-degenerate triangles
template <class Tri>
__device__ __forceinline__ void cell_walk(const Cell& c, const Node& nd, Tri&& tri) {
    unsigned left = c.em;
    while (left) {
        const int r = __ffs(left) - 1;
        int prev = c.nxt[r];
        left &= ~((1u << r) | (1u << prev));
        int cur = c.nxt[prev];
        while (cur != r) {
            if (!same_pos(c, r, prev, nd) && !same_pos(c, prev, cur, nd) && !same_pos(c, r, cur, nd)) tri(r, prev, cur);
            left &= ~(1u << cur);
            prev = cur;
            cur = c.nxt[cur];
        }
    }
}

// loads the 8 corners of the cell at nd (when it has one) and returns its inside bits, or 0 / 255 for an empty cell
__device__ __forceinline__ unsigned load_cell(const float* __restrict__ vol, const Node& nd, int d0, int d1, int d2, float level,
                                              Cell& c) {
    if (nd.a + 1 >= d0 || nd.b + 1 >= d1 || nd.c + 1 >= d2) return 0u;
    const long long s0 = (long long)d1 * d2, s1 = d2;
    unsigned ins = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        c.cv[k] = __ldg(vol + nd.n + ((k >> 2) & 1) * s0 + ((k >> 1) & 1) * s1 + (k & 1));
        ins |= (c.cv[k] > level ? 1u : 0u) << k;
    }
    return ins;
}

// sign-change edges of a node along +a, +b, +c (bit axis)
__device__ __forceinline__ unsigned node_edges(const float* __restrict__ vol, long long n, int a, int b, int c, int d0, int d1,
                                               int d2, float level) {
    const long long s0 = (long long)d1 * d2, s1 = d2;
    const bool in0 = __ldg(vol + n) > level;
    unsigned m = 0;
    if (a + 1 < d0 && ((__ldg(vol + n + s0) > level) != in0)) m |= 1u;
    if (b + 1 < d1 && ((__ldg(vol + n + s1) > level) != in0)) m |= 2u;
    if (c + 1 < d2 && ((__ldg(vol + n + 1) > level) != in0)) m |= 4u;
    return m;
}

__global__ void __launch_bounds__(kThreads) k_mc_count(const float* __restrict__ vol, int d0, int d1, int d2, float level,
                                                       unsigned long long* __restrict__ scan, unsigned long long* totals) {
    const long long nn = (long long)d0 * d1 * d2;
    const long long n = (long long)blockIdx.x * kThreads + threadIdx.x;
    unsigned nv = 0, nt = 0;
    if (n < nn) {
        const Node nd = node_of(n, d1, d2);
        nv = __popc(node_edges(vol, n, nd.a, nd.b, nd.c, d0, d1, d2, level));
        Cell c;
        const unsigned ins = load_cell(vol, nd, d0, d1, d2, level, c);
        if (ins != 0u && ins != 255u) {
            cell_build(c, ins, level);
            cell_walk(c, nd, [&](int, int, int) { ++nt; });
        }
        scan[n] = (unsigned long long)nv | ((unsigned long long)nt << 32);
    }
    // exact 64-bit totals (the scan's high word may wrap for absurd sizes; p3d_mc_emit refuses those)
    __shared__ unsigned long long s_v[kThreads / 32], s_t[kThreads / 32];
    unsigned long long v = nv, t = nt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v += __shfl_xor_sync(0xffffffffu, v, o);
        t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = v; s_t[threadIdx.x >> 5] = t; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long sv = 0, st = 0;
        for (int w = 0; w < kThreads / 32; ++w) { sv += s_v[w]; st += s_t[w]; }
        if (sv) atomicAdd(totals, sv);
        if (st) atomicAdd(totals + 1, st);
    }
}

// gradient component along one axis at a node: central difference inside, one-sided at the border
__device__ __forceinline__ float grad_at(const float* __restrict__ vol, long long n, int i, int D, long long stride) {
    if (i == 0) return __fsub_rn(__ldg(vol + n + stride), __ldg(vol + n));
    if (i == D - 1) return __fsub_rn(__ldg(vol + n), __ldg(vol + n - stride));
    return __fmul_rn(__fsub_rn(__ldg(vol + n + stride), __ldg(vol + n - stride)), 0.5f);
}

struct EmitArgs {
    const float* vol;
    int d0, d1, d2;
    float level;
    const unsigned long long *scan, *totals;
    float* verts;
    int* faces;
    float *normals, *values;
    long long* floor_node;
};

__device__ __forceinline__ void write_vertex(const EmitArgs& A, const Node& nd, int ax, long long idx) {
    const long long s[3] = {(long long)A.d1 * A.d2, (long long)A.d2, 1};
    const int D[3] = {A.d0, A.d1, A.d2};
    const float vlo = __ldg(A.vol + nd.n), vhi = __ldg(A.vol + nd.n + s[ax]);
    const float t = __fdiv_rn(__fsub_rn(A.level, vlo), __fsub_rn(vhi, vlo));
    const int lo[3] = {nd.a, nd.b, nd.c};
    float p[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) p[d] = d == ax ? __fadd_rn((float)lo[d], t) : (float)lo[d];
#pragma unroll
    for (int d = 0; d < 3; ++d) A.verts[idx * 3 + d] = p[d];
    if (A.values) A.values[idx] = fmaxf(vlo, vhi);
    if (A.floor_node) {
        const long long fa = (long long)floorf(p[0]), fb = (long long)floorf(p[1]), fc = (long long)floorf(p[2]);
        A.floor_node[idx] = (fa * A.d1 + fb) * A.d2 + fc;
    }
    if (A.normals) {
        float g[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const int ilo = lo[d], ihi = lo[d] + (d == ax ? 1 : 0);
            const float glo = grad_at(A.vol, nd.n, ilo, D[d], s[d]);
            const float ghi = grad_at(A.vol, nd.n + s[ax], ihi, D[d], s[d]);
            g[d] = -__fadd_rn(glo, __fmul_rn(t, __fsub_rn(ghi, glo)));       // descent: towards lower density
        }
        const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2])));
#pragma unroll
        for (int d = 0; d < 3; ++d) A.normals[idx * 3 + d] = len > 0.f ? __fdiv_rn(g[d], len) : 0.f;
    }
}

// global index of the vertex on local edge e: the owner node's scanned offset + its sign-change edges along lower axes
__device__ __forceinline__ int vertex_id(const EmitArgs& A, const Node& nd, const Cell& c, int e) {
    const int k = kEdgeCorner[e], ax = kEdgeAxis[e];
    const int oa = nd.a + ((k >> 2) & 1), ob = nd.b + ((k >> 1) & 1);
    const long long s0 = (long long)A.d1 * A.d2, s1 = A.d2;
    const long long o = nd.n + ((k >> 2) & 1) * s0 + ((k >> 1) & 1) * s1 + (k & 1);
    int id = (int)(unsigned)A.scan[o];
    const bool in0 = c.cv[k] > A.level;
    if (ax >= 1 && oa + 1 < A.d0) id += (__ldg(A.vol + o + s0) > A.level) != in0;
    if (ax >= 2 && ob + 1 < A.d1) id += (__ldg(A.vol + o + s1) > A.level) != in0;
    return id;
}

__global__ void __launch_bounds__(kThreads) k_mc_emit(const EmitArgs A) {
    if (A.totals[0] >= (1ull << 31) || A.totals[1] >= (1ull << 31)) return;       // faces are int32
    const long long nn = (long long)A.d0 * A.d1 * A.d2;
    const long long n = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (n >= nn) return;
    const Node nd = node_of(n, A.d1, A.d2);
    const unsigned long long packed = A.scan[n];
    const unsigned m = node_edges(A.vol, n, nd.a, nd.b, nd.c, A.d0, A.d1, A.d2, A.level);
    long long vi = (long long)(unsigned)packed;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax)
        if (m & (1u << ax)) write_vertex(A, nd, ax, vi++);
    Cell c;
    const unsigned ins = load_cell(A.vol, nd, A.d0, A.d1, A.d2, A.level, c);
    if (ins == 0u || ins == 255u) return;
    cell_build(c, ins, A.level);
    long long ti = (long long)(packed >> 32);
    cell_walk(c, nd, [&](int e0, int e1, int e2) {
        A.faces[ti * 3 + 0] = vertex_id(A, nd, c, e0);
        A.faces[ti * 3 + 1] = vertex_id(A, nd, c, e1);
        A.faces[ti * 3 + 2] = vertex_id(A, nd, c, e2);
        ++ti;
    });
}

__global__ void __launch_bounds__(kThreads) k_mc_lattice(const long long* __restrict__ flat, long long n_points, int R, float vsize,
                                                         float vorigin, float* __restrict__ coords) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n_points) return;
    float x, y, z;
    dev::volume_point(dev::volume_dest(flat[i], R), R, vsize, vorigin, x, y, z);
    coords[i * 3 + 0] = x; coords[i * 3 + 1] = y; coords[i * 3 + 2] = z;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int check_dims(int64_t d0, int64_t d1, int64_t d2) {
    P3D_REQUIRE(d0 >= 2 && d1 >= 2 && d2 >= 2, "marching cubes needs every volume side >= 2, got (%lld, %lld, %lld)",
                (long long)d0, (long long)d1, (long long)d2);
    // every factor is bounded before it is multiplied: products of unchecked int64 sides wrap (2 * 2 * (2^62 + 1) == 4)
    P3D_REQUIRE(d0 <= kMaxNodes && d1 <= kMaxNodes && d2 <= kMaxNodes && d0 * d1 <= kMaxNodes && d0 * d1 * d2 <= kMaxNodes,
                "marching cubes supports at most 2^30 nodes, got (%lld, %lld, %lld)", (long long)d0, (long long)d1, (long long)d2);
    return P3D_OK;
}

int scan_temp_bytes(long long nn, size_t* bytes) {
    P3D_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, *bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)nn));
    return P3D_OK;
}

}  // namespace

}  // namespace p3d

using namespace p3d;

extern "C" {

size_t p3d_mc_workspace_bytes(int64_t d0, int64_t d1, int64_t d2) {
    if (check_dims(d0, d1, d2)) return 0;
    const long long nn = d0 * d1 * d2;
    size_t temp = 0;
    if (scan_temp_bytes(nn, &temp)) return 0;
    return kHead + align256((size_t)nn * 8) + align256(temp);
}

int p3d_mc_count(const float* vol, int64_t d0, int64_t d1, int64_t d2, float level, void* workspace, size_t workspace_bytes,
                 int64_t* counts2, void* stream) {
    int rc = check_dims(d0, d1, d2);
    if (rc) return rc;
    P3D_REQUIRE(vol && workspace && counts2, "null pointer");
    const long long nn = d0 * d1 * d2;
    size_t temp = 0;
    if ((rc = scan_temp_bytes(nn, &temp))) return rc;
    const size_t need = kHead + align256((size_t)nn * 8) + align256(temp);
    if (workspace_bytes < need) { set_error("marching cubes workspace too small: need %zu bytes, got %zu", need, workspace_bytes); return P3D_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    auto* totals = reinterpret_cast<unsigned long long*>(ws);
    auto* scan = reinterpret_cast<unsigned long long*>(ws + kHead);
    P3D_CUDA_TRY(cudaMemsetAsync(totals, 0, 2 * sizeof(unsigned long long), st));
    {
        ProfileScope prof(PROF_OTHER, st);
        k_mc_count<<<(unsigned)((nn + kThreads - 1) / kThreads), kThreads, 0, st>>>(vol, (int)d0, (int)d1, (int)d2, level, scan, totals);
        P3D_LAUNCH_CHECK();
        P3D_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + kHead + align256((size_t)nn * 8), temp, scan, scan, (int)nn, st));
        count_launch(2);                                  // CUB's scan: init + scan kernels
    }
    P3D_CUDA_TRY(cudaMemcpyAsync(counts2, totals, 2 * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return P3D_OK;
}

int p3d_mc_emit(const float* vol, int64_t d0, int64_t d1, int64_t d2, float level, const void* workspace, size_t workspace_bytes,
                float* verts, int32_t* faces, float* normals, float* values, int64_t* floor_node, void* stream) {
    int rc = check_dims(d0, d1, d2);
    if (rc) return rc;
    P3D_REQUIRE(vol && workspace && verts && faces, "null pointer");
    const long long nn = d0 * d1 * d2;
    P3D_REQUIRE(workspace_bytes >= kHead + (size_t)nn * 8, "marching cubes workspace too small (pass the one of p3d_mc_count)");
    const unsigned char* ws = reinterpret_cast<const unsigned char*>(workspace);
    EmitArgs a;
    a.vol = vol; a.d0 = (int)d0; a.d1 = (int)d1; a.d2 = (int)d2; a.level = level;
    a.totals = reinterpret_cast<const unsigned long long*>(ws);
    a.scan = reinterpret_cast<const unsigned long long*>(ws + kHead);
    a.verts = verts; a.faces = faces; a.normals = normals; a.values = values;
    a.floor_node = reinterpret_cast<long long*>(floor_node);
    cudaStream_t st = (cudaStream_t)stream;
    ProfileScope prof(PROF_OTHER, st);
    k_mc_emit<<<(unsigned)((nn + kThreads - 1) / kThreads), kThreads, 0, st>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

int p3d_mc_lattice_coords(const int64_t* flat, int64_t n_points, int32_t resolution, double cube_length, float* coords, void* stream) {
    P3D_REQUIRE(resolution >= 2 && cube_length > 0 && n_points >= 0, "bad arguments");
    if (n_points == 0) return P3D_OK;
    P3D_REQUIRE(flat && coords, "null pointer");
    const float vsize = (float)(cube_length / (double)(resolution - 1));     // as p3d_volume_query rounds them
    const float vorigin = (float)(0.0 - cube_length / 2.0);
    cudaStream_t st = (cudaStream_t)stream;
    k_mc_lattice<<<(unsigned)((n_points + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        reinterpret_cast<const long long*>(flat), n_points, resolution, vsize, vorigin, coords);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // extern "C"
