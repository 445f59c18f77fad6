// Marching cubes over a dense fp32 grid (the mesh renderer's density cube, if_mesh_renderer.py:42-48).
//
// nb_mcubes_count: one thread per grid point p = (i, j, k) (k fastest, so neighbouring threads read neighbouring
// values).  p owns the edges p -> p + e_x / e_y / e_z and is the min corner of one cell; it writes a 16-bit code =
// crossing mask (3 bits) | cell case << 3.  Two CUB exclusive scans turn the per-point vertex counts (popcount of the
// mask) and triangle counts (nb_mc_num_tris[case]) into output offsets, and the totals go to counts[2].
// nb_mcubes_emit (after the caller read the totals and allocated): the same threads write their vertices and
// triangles at those offsets.  No atomics: the output order is the grid order, so the mesh is deterministic.
//
// nb_mesh_inside (the multi-view mesh dataset's prepare_inside_pts, float32 camera): mesh_inside_kernel<float> of
// nb_mesh_inside.cuh.
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "nb_mesh_inside.cuh"

#define NB_MC_TABLE_QUALIFIER static __constant__
#include "nb_mc_table.h"

namespace nb {
namespace {

constexpr int kMcThreads = 256;

struct McGrid {
    const float* v;
    int nx, ny, nz;
    long long n;            // points
    double iso;
    int has_cells;          // all dims >= 2: otherwise there is no cell and hence no surface
};

__device__ __forceinline__ bool inside(float x, double iso) { return (double)x > iso; }

__host__ __device__ __forceinline__ int popc3(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1); }

struct VertCount {
    __host__ __device__ int operator()(uint16_t c) const { return popc3(c & 7); }
};
struct TriCount {
    __device__ int operator()(uint16_t c) const { return nb_mc_num_tris[c >> 3]; }
};

// code of every point; code[n] = 0 so that an exclusive scan over n + 1 entries ends with the totals
__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(McGrid g, uint16_t* __restrict__ code) {
    const long long p = (long long)blockIdx.x * kMcThreads + threadIdx.x;
    if (p > g.n) return;
    if (p == g.n || !g.has_cells) { code[p] = 0; return; }
    const long long sy = g.nz, sx = (long long)g.ny * g.nz;
    const int k = (int)(p % g.nz), j = (int)((p / g.nz) % g.ny), i = (int)(p / sx);
    const float* v = g.v + p;
    const bool in0 = inside(__ldg(v), g.iso);
    const bool hx = i + 1 < g.nx, hy = j + 1 < g.ny, hz = k + 1 < g.nz;
    int mask = 0;
    if (hx && inside(__ldg(v + sx), g.iso) != in0) mask |= 1;
    if (hy && inside(__ldg(v + sy), g.iso) != in0) mask |= 2;
    if (hz && inside(__ldg(v + 1), g.iso) != in0) mask |= 4;
    int cs = 0;
    if (hx && hy && hz) {
        cs = in0 ? 1 : 0;
#pragma unroll
        for (int c = 1; c < 8; ++c) {
            const long long off = (c & 1 ? sx : 0) + (c & 2 ? sy : 0) + (c & 4 ? 1 : 0);
            cs |= (inside(__ldg(v + off), g.iso) ? 1 : 0) << c;
        }
    }
    code[p] = (uint16_t)(mask | (cs << 3));
}

__global__ void mc_totals_kernel(const int* __restrict__ vert_off, const int* __restrict__ tri_off, long long n,
                                 long long* __restrict__ counts) {
    counts[0] = vert_off[n];
    counts[1] = tri_off[n];
}

__global__ void __launch_bounds__(kMcThreads) mc_emit_kernel(McGrid g, const uint16_t* __restrict__ code,
                                                             const int* __restrict__ vert_off, const int* __restrict__ tri_off,
                                                             double* __restrict__ verts, long long* __restrict__ tris) {
    const long long p = (long long)blockIdx.x * kMcThreads + threadIdx.x;
    if (p >= g.n) return;
    const int c = code[p];
    if (c == 0) return;
    const long long sy = g.nz, sx = (long long)g.ny * g.nz;
    const int k = (int)(p % g.nz), j = (int)((p / g.nz) % g.ny), i = (int)(p / sx);
    const int mask = c & 7;
    if (mask) {
        const double f0 = (double)__ldg(g.v + p);
        double* out = verts + (size_t)vert_off[p] * 3;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (!(mask >> a & 1)) continue;
            const double f1 = (double)__ldg(g.v + p + (a == 0 ? sx : a == 1 ? sy : 1));
            const double t = (g.iso - f0) / (f1 - f0);     // fp64, as the reference's float64 cube is interpolated
            out[0] = (double)i + (a == 0 ? t : 0.0);
            out[1] = (double)j + (a == 1 ? t : 0.0);
            out[2] = (double)k + (a == 2 ? t : 0.0);
            out += 3;
        }
    }
    const int cs = c >> 3;
    const int nt = nb_mc_num_tris[cs];
    long long* out = tris + (size_t)tri_off[p] * 3;
    for (int e = 0; e < 3 * nt; ++e) {
        const int edge = nb_mc_tris[cs][e];
        const int ax = nb_mc_edge_axis[edge];
        const long long q = p + nb_mc_edge_offset[edge][0] * sx + nb_mc_edge_offset[edge][1] * sy + nb_mc_edge_offset[edge][2];
        const int m = code[q] & 7;
        out[e] = (long long)vert_off[q] + popc3(m & ((1 << ax) - 1));
    }
}

// workspace layout: code (n + 1) u16 | vert_off (n + 1) i32 | tri_off (n + 1) i32 | CUB scratch, 256-byte aligned each
struct McLayout {
    size_t code, vert_off, tri_off, scratch, scratch_bytes, total;
};

int mc_layout(long long n, McLayout* L) {
    const int items = (int)(n + 1);
    size_t sv = 0, st = 0;
    auto vin = thrust::make_transform_iterator((const uint16_t*)nullptr, VertCount());
    auto tin = thrust::make_transform_iterator((const uint16_t*)nullptr, TriCount());
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, sv, vin, (int*)nullptr, items);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, st, tin, (int*)nullptr, items);
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("nb_mcubes: scan size query failed: %s", cudaGetErrorString(e));
        return NB_ERR_CUDA;
    }
    L->code = 0;
    L->vert_off = align256(L->code + (size_t)(n + 1) * sizeof(uint16_t));
    L->tri_off = align256(L->vert_off + (size_t)(n + 1) * sizeof(int));
    L->scratch = align256(L->tri_off + (size_t)(n + 1) * sizeof(int));
    L->scratch_bytes = sv > st ? sv : st;
    L->total = align256(L->scratch + L->scratch_bytes);
    return NB_OK;
}

// shared validation of count / emit: null pointers, dims, the 32-bit offset limit, workspace size
int mc_check(const nb_mcubes_args* a, const char* who, McGrid* g, McLayout* L) {
    if (!a || !a->grid || !a->workspace || !a->counts) { set_error("%s: null argument", who); return NB_ERR_BAD_ARG; }
    if (a->nx < 1 || a->ny < 1 || a->nz < 1) { set_error("%s: grid dims must be >= 1 (got %d x %d x %d)", who, a->nx, a->ny, a->nz); return NB_ERR_BAD_ARG; }
    const long long n = (long long)a->nx * a->ny * a->nz;
    const long long cells = (long long)(a->nx - 1) * (a->ny - 1) * (a->nz - 1);
    if (5 * cells >= (1LL << 31) || 3 * n >= (1LL << 31)) {
        set_error("%s: a %d x %d x %d grid exceeds the 32-bit offsets (5 * cells and 3 * points must stay below 2^31)",
                  who, a->nx, a->ny, a->nz);
        return NB_ERR_UNSUPPORTED;
    }
    const int st = mc_layout(n, L);
    if (st != NB_OK) return st;
    if (a->workspace_bytes < L->total) { set_error("%s: workspace_bytes too small (%zu < %zu)", who, a->workspace_bytes, L->total); return NB_ERR_BAD_ARG; }
    g->v = a->grid; g->nx = a->nx; g->ny = a->ny; g->nz = a->nz; g->n = n; g->iso = a->isovalue;
    g->has_cells = cells > 0;
    return NB_OK;
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_mcubes_workspace_bytes(int nx, int ny, int nz) {
    if (nx < 1 || ny < 1 || nz < 1 || 3LL * nx * ny * nz >= (1LL << 31)) return 0;
    McLayout L;
    return mc_layout((long long)nx * ny * nz, &L) == NB_OK ? L.total : 0;
}

int nb_mcubes_count(const nb_mcubes_args* a, void* stream) {
    McGrid g;
    McLayout L;
    const int chk = mc_check(a, "nb_mcubes_count", &g, &L);
    if (chk != NB_OK) return chk;
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)a->workspace;
    uint16_t* code = (uint16_t*)(ws + L.code);
    int* vert_off = (int*)(ws + L.vert_off);
    int* tri_off = (int*)(ws + L.tri_off);
    const long long items = g.n + 1;
    mc_count_kernel<<<(unsigned)((items + kMcThreads - 1) / kMcThreads), kMcThreads, 0, st>>>(g, code);
    size_t sb = L.scratch_bytes;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(ws + L.scratch, sb, thrust::make_transform_iterator((const uint16_t*)code, VertCount()),
                                                  vert_off, (int)items, st);
    if (e == cudaSuccess) {
        sb = L.scratch_bytes;
        e = cub::DeviceScan::ExclusiveSum(ws + L.scratch, sb, thrust::make_transform_iterator((const uint16_t*)code, TriCount()),
                                          tri_off, (int)items, st);
    }
    if (e == cudaSuccess) {
        mc_totals_kernel<<<1, 1, 0, st>>>(vert_off, tri_off, g.n, a->counts);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("nb_mcubes_count: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_mcubes_emit(const nb_mcubes_args* a, void* stream) {
    McGrid g;
    McLayout L;
    const int chk = mc_check(a, "nb_mcubes_emit", &g, &L);
    if (chk != NB_OK) return chk;
    if (!a->vertices || !a->triangles) { set_error("nb_mcubes_emit: null vertices / triangles (skip the call for an empty mesh)"); return NB_ERR_BAD_ARG; }
    char* ws = (char*)a->workspace;
    mc_emit_kernel<<<(unsigned)((g.n + kMcThreads - 1) / kMcThreads), kMcThreads, 0, (cudaStream_t)stream>>>(
        g, (const uint16_t*)(ws + L.code), (const int*)(ws + L.vert_off), (const int*)(ws + L.tri_off), a->vertices, a->triangles);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_mcubes_emit: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_mesh_inside(const nb_mesh_inside_args* a, void* stream) {
    if (!a || !a->x || !a->y || !a->z || !a->msks || !a->RT || !a->Ks || !a->inside) {
        set_error("nb_mesh_inside: null argument");
        return NB_ERR_BAD_ARG;
    }
    return mesh_inside_launch<float>("nb_mesh_inside", a, a->RT, a->Ks, stream);
}

}  // extern "C"
