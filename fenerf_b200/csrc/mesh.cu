// Marching cubes over a dense density grid (fenerf_mc_*): the mesh the shape scripts leave to the CPU
// (extract_double_semantic_shapes.py writes the 256^3 grid to an .mrc file for skimage's mesher).
//
//   classify      one thread per grid point: the case index of the cell whose lowest corner it is, and which of the three
//                 edges it owns (+axis 0, +axis 1, +axis 2 from the point) sigma crosses `level` on; the vertex and triangle
//                 counts go into the arrays the scans turn into offsets, their totals into two int64 counters
//   scans         exclusive sums of both counts (CUB), in place, over N^3 + 1 entries: the last holds the total
//   emit_vertices one vertex per owned crossed edge, at vertex_offset[owner] + its rank among the owner's crossed edges
//   emit_faces    one thread per cell, its table triangles at triangle_offset[cell]; each edge's vertex index is found
//                 from its owner's offset and flags, so no vertex is written twice and the order is fixed
// The tables come from tools/gen_mc_tables.py (mc_tables.h); DESIGN.md section 10 describes them.
#include "common.cuh"
#include "mc_tables.h"

#include <cub/device/device_scan.cuh>
#include <math.h>

namespace fn {
namespace {

constexpr int kBlock = 256;
constexpr long long kMaxPoints = 2147483646LL;    // N^3 + 1 scan entries in an int

struct McWorkspace {
    size_t cube, edges, voff, toff, scan, scan_bytes, total;
};

McWorkspace plan(int n) {
    const size_t pts = (size_t)n * n * n;
    McWorkspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = fn_align_up(off + bytes, 256); return o; };
    w.cube = take(pts);
    w.edges = take(pts);
    w.voff = take((pts + 1) * 4);
    w.toff = take((pts + 1) * 4);
    w.scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, w.scan_bytes, (int*)nullptr, (int)(pts + 1));
    w.scan = take(w.scan_bytes);
    w.total = off;
    return w;
}

__device__ __forceinline__ bool inside(float s, float level) { return s >= level; }    // NaN: outside

__global__ void __launch_bounds__(kBlock) mc_classify_kernel(const float* __restrict__ sigma, int n, float level,
                                                             uint8_t* __restrict__ cube, uint8_t* __restrict__ edges,
                                                             int* __restrict__ vcount, int* __restrict__ tcount,
                                                             unsigned long long* __restrict__ totals) {
    __shared__ uint8_t tri_count[256];
    __shared__ unsigned long long part[2][kBlock / 32];
    for (int c = threadIdx.x; c < 256; c += blockDim.x) tri_count[c] = kMcTriCount[c];
    __syncthreads();
    const long long nn = (long long)n * n, pts = nn * n;
    const long long stride[3] = {nn, n, 1};
    unsigned long long nv = 0, nt = 0;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pts; p += (long long)gridDim.x * blockDim.x) {
        const int idx[3] = {(int)(p / nn), (int)(p / n % n), (int)(p % n)};
        const bool in0 = inside(sigma[p], level);
        unsigned flags = 0;
        for (int a = 0; a < 3; ++a)
            if (idx[a] < n - 1 && inside(sigma[p + stride[a]], level) != in0) flags |= 1u << a;
        unsigned c = 0;
        if (idx[0] < n - 1 && idx[1] < n - 1 && idx[2] < n - 1) {
            c = in0 ? 1u : 0u;
            for (int k = 1; k < 8; ++k) {
                const long long q = p + (k & 1) * stride[0] + ((k >> 1) & 1) * stride[1] + ((k >> 2) & 1) * stride[2];
                c |= (inside(sigma[q], level) ? 1u : 0u) << k;
            }
        }
        const int v = __popc(flags), t = tri_count[c];
        cube[p] = (uint8_t)c;
        edges[p] = (uint8_t)flags;
        vcount[p] = v;
        tcount[p] = t;
        nv += v;
        nt += t;
    }
    for (int o = 16; o > 0; o >>= 1) {
        nv += __shfl_down_sync(0xffffffffu, nv, o);
        nt += __shfl_down_sync(0xffffffffu, nt, o);
    }
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane == 0) { part[0][warp] = nv; part[1][warp] = nt; }
    __syncthreads();
    if (threadIdx.x < 2) {
        unsigned long long s = 0;
        for (int w = 0; w < kBlock / 32; ++w) s += part[threadIdx.x][w];
        if (s) atomicAdd(totals + threadIdx.x, s);           // integers: the totals do not depend on the order
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { vcount[pts] = 0; tcount[pts] = 0; }
}

// the lattice coordinate origin + i * voxel, rounded as the density grid's points are (a product, then a sum)
__device__ __forceinline__ float lattice(float origin, int i, float voxel) { return __fadd_rn(__fmul_rn((float)i, voxel), origin); }

__global__ void __launch_bounds__(kBlock) mc_emit_vertices_kernel(const float* __restrict__ sigma, int n, float level,
                                                                  float ox, float oy, float oz, float voxel,
                                                                  const uint8_t* __restrict__ edges,
                                                                  const int* __restrict__ voff, long long nv,
                                                                  float* __restrict__ verts) {
    const long long nn = (long long)n * n, pts = nn * n;
    const long long stride[3] = {nn, n, 1};
    const float origin[3] = {ox, oy, oz};
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pts; p += (long long)gridDim.x * blockDim.x) {
        const unsigned flags = edges[p];
        if (!flags) continue;
        const int idx[3] = {(int)(p / nn), (int)(p / n % n), (int)(p % n)};
        float base[3];
        for (int a = 0; a < 3; ++a) base[a] = lattice(origin[a], idx[a], voxel);
        const float sa = sigma[p];
        long long v = voff[p];
        for (int a = 0; a < 3; ++a) {
            if (!((flags >> a) & 1)) continue;
            const float sb = sigma[p + stride[a]];
            float t = __fdiv_rn(__fsub_rn(level, sa), __fsub_rn(sb, sa));
            if (!(t >= 0.f && t <= 1.f)) t = 0.5f;             // a NaN or infinite end: the edge's midpoint
            const float b = lattice(origin[a], idx[a] + 1, voxel);
            if (v >= nv) return;                                   // a caller's count below fenerf_mc_count's
            float* out = verts + 3 * v++;
            for (int d = 0; d < 3; ++d) out[d] = base[d];
            out[a] = __fmaf_rn(t, __fsub_rn(b, base[a]), base[a]);
        }
    }
}

__global__ void __launch_bounds__(kBlock) mc_emit_faces_kernel(int n, const uint8_t* __restrict__ cube,
                                                               const uint8_t* __restrict__ edges, const int* __restrict__ voff,
                                                               const int* __restrict__ toff, long long nt,
                                                               int* __restrict__ faces) {
    __shared__ uint8_t tris[256][FN_MC_MAX_TRIS * 3];
    __shared__ uint8_t tri_count[256];
    __shared__ long long edge_step[12];
    __shared__ uint8_t edge_axis[12];
    const long long nn = (long long)n * n, pts = nn * n;
    for (int i = threadIdx.x; i < 256 * FN_MC_MAX_TRIS * 3; i += blockDim.x) (&tris[0][0])[i] = (&kMcTris[0][0])[i];
    for (int c = threadIdx.x; c < 256; c += blockDim.x) tri_count[c] = kMcTriCount[c];
    if (threadIdx.x < 12) {
        const int c0 = kMcEdgeCorner[threadIdx.x];
        edge_step[threadIdx.x] = (c0 & 1) * nn + ((c0 >> 1) & 1) * n + ((c0 >> 2) & 1);
        edge_axis[threadIdx.x] = kMcEdgeAxis[threadIdx.x];
    }
    __syncthreads();
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pts; p += (long long)gridDim.x * blockDim.x) {
        const int c = cube[p];
        const int cnt = tri_count[c];
        if (!cnt || toff[p] + cnt > nt) continue;
        int* out = faces + 3 * (long long)toff[p];
        for (int i = 0; i < 3 * cnt; ++i) {
            const int e = tris[c][i];
            const long long q = p + edge_step[e];
            const unsigned below = edges[q] & ((1u << edge_axis[e]) - 1u);
            out[i] = voff[q] + __popc(below);
        }
    }
}

int blocks_for(long long n) {
    long long want = (n + kBlock - 1) / kBlock, cap = (long long)num_sms() * 16;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

// a device (or managed) pointer of the current context; host memory, registered or not, is refused
int require_device(const void* p, const char* name) {
    FN_REQUIRE(p, "%s is NULL", name);
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return fail(FENERF_E_ARG, "%s is not a CUDA pointer", name);
    }
    FN_REQUIRE(attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged,
               "%s is a host pointer: the marching cubes run on the device only", name);
    return 0;
}

int check_grid(const float* sigma, int n, float level, void* workspace, size_t workspace_bytes) {
    FN_REQUIRE(n >= 2, "grid side N = %d: a mesh needs N >= 2", n);
    FN_REQUIRE((long long)n * n * n + 1 <= kMaxPoints, "grid side N = %d: N^3 + 1 grid points exceed 2^31 - 1", n);
    FN_REQUIRE(isfinite(level), "level must be finite");
    if (int e = require_device(sigma, "sigma")) return e;
    if (int e = require_device(workspace, "workspace")) return e;
    FN_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    const size_t need = plan(n).total;
    if (workspace_bytes < need) return fail(FENERF_E_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, need);
    return 0;
}

}  // namespace
}  // namespace fn

using namespace fn;

extern "C" {
#pragma GCC visibility push(default)

size_t fenerf_mc_workspace_bytes(int32_t n) {
    if (n < 2 || (long long)n * n * n + 1 > kMaxPoints) return 0;
    return plan(n).total;
}

int fenerf_mc_count(const float* sigma, int32_t n, float level, void* workspace, size_t workspace_bytes, int64_t* counts,
                    void* stream) {
    if (int e = check_grid(sigma, n, level, workspace, workspace_bytes)) return e;
    if (int e = require_device(counts, "counts")) return e;
    FN_REQUIRE(((uintptr_t)counts & 7) == 0, "counts must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const McWorkspace w = plan(n);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    const long long pts = (long long)n * n * n;
    int* voff = reinterpret_cast<int*>(ws + w.voff);
    int* toff = reinterpret_cast<int*>(ws + w.toff);
    FN_CUDA_OK(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), st));
    if (int e = launch<mc_classify_kernel>("mc_classify_kernel", blocks_for(pts), kBlock, 0, st, sigma, (int)n, level,
                                           ws + w.cube, ws + w.edges, voff, toff,
                                           reinterpret_cast<unsigned long long*>(counts)))
        return e;
    // the sums wrap for a mesh past 2^31 - 1 vertices or triangles; fenerf_mc_emit refuses those from the exact totals
    for (int* a : {voff, toff}) {
        size_t bytes = w.scan_bytes;
        FN_CUDA_OK(cub::DeviceScan::ExclusiveSum(ws + w.scan, bytes, a, (int)(pts + 1), st));
        FN_LAUNCH_OK("cub::DeviceScan::ExclusiveSum");
    }
    return 0;
}

int fenerf_mc_emit(const float* sigma, int32_t n, float level, const float* origin, float voxel_size, const void* workspace,
                   size_t workspace_bytes, int64_t n_vertices, int64_t n_triangles, float* vertices, int32_t* faces,
                   void* stream) {
    if (int e = check_grid(sigma, n, level, const_cast<void*>(workspace), workspace_bytes)) return e;
    FN_REQUIRE(origin, "origin is NULL");
    FN_REQUIRE(n_vertices >= 0 && n_triangles >= 0, "negative counts");
    FN_REQUIRE(n_vertices <= 2147483647LL && n_triangles <= 2147483647LL,
               "%lld vertices and %lld triangles: more than 2^31 - 1 do not fit the int32 indices",
               (long long)n_vertices, (long long)n_triangles);
    if (n_vertices) if (int e = require_device(vertices, "vertices")) return e;
    if (n_triangles) if (int e = require_device(faces, "faces")) return e;
    cudaStream_t st = (cudaStream_t)stream;
    const McWorkspace w = plan(n);
    const unsigned char* ws = static_cast<const unsigned char*>(workspace);
    const long long pts = (long long)n * n * n;
    const int* voff = reinterpret_cast<const int*>(ws + w.voff);
    const int* toff = reinterpret_cast<const int*>(ws + w.toff);
    if (n_vertices)
        if (int e = launch<mc_emit_vertices_kernel>("mc_emit_vertices_kernel", blocks_for(pts), kBlock, 0, st, sigma, (int)n,
                                                    level, origin[0], origin[1], origin[2], voxel_size, ws + w.edges, voff,
                                                    (long long)n_vertices, vertices))
            return e;
    if (n_triangles)
        if (int e = launch<mc_emit_faces_kernel>("mc_emit_faces_kernel", blocks_for(pts), kBlock, 0, st, (int)n, ws + w.cube,
                                                 ws + w.edges, voff, toff, (long long)n_triangles, faces))
            return e;
    return 0;
}

#pragma GCC visibility pop
}  // extern "C"
