// The mesh datasets' prepare_inside_pts on the device: one thread per world-grid point, k fastest; the point is built from
// the three axis arrays and projected into the mask views with the masked renderers' projection (nb_device.cuh).
// mesh_inside_kernel is instantiated over the camera's scalar type: float for nb_mesh_inside (nb_mcubes.cu, the
// multi-view dataset's float32 camera) and double for nb_mesh_inside_f64 (nb_mesh_inside_f64.cu, the monocular dataset's
// float64 camera).  Each translation unit instantiates one, so each object holds exactly one mesh_inside_kernel.
#pragma once

#include "nb_device.cuh"

namespace nb {
namespace {

constexpr int kInsideThreads = 256;

template <typename T>
struct InsideGrid {
    const float *x, *y, *z;
    unsigned ny, nz, n;         // n <= 2^31, so a point index fits in 32 bits
    const unsigned char* msks;
    const T *RT, *Ks;
    int nv, H, W;
    unsigned char* inside;
};

template <typename T>
__global__ void __launch_bounds__(kInsideThreads) mesh_inside_kernel(const __grid_constant__ InsideGrid<T> g) {
    const unsigned p = blockIdx.x * kInsideThreads + threadIdx.x;
    if (p >= g.n) return;
    const unsigned nyz = g.ny * g.nz;
    const unsigned i = p / nyz, r = p - i * nyz, j = r / g.nz, k = r - j * g.nz;
    const float wx = __ldg(g.x + i), wy = __ldg(g.y + j), wz = __ldg(g.z + k);
    unsigned char val = 1;
    for (int v = 0; v < g.nv && val == 1; ++v) {
        T ix, iy, iz;
        project_view(g.RT + v * 12, g.Ks + v * 9, wx, wy, wz, ix, iy, iz);
        const int u = mask_pixel_i32(div_rn(ix, iz), g.W), w = mask_pixel_i32(div_rn(iy, iz), g.H);
        val = __ldg(g.msks + ((size_t)v * g.H + w) * g.W + u);
    }
    g.inside[p] = val;
}

// Validation of everything but the pointers (the callers check those: the two entry points take the camera from different
// places), then one launch.  Nothing is enqueued unless every check passes.
template <typename T>
int mesh_inside_launch(const char* who, const nb_mesh_inside_args* a, const T* RT, const T* Ks, void* stream) {
    if (a->nv < 1 || a->H < 1 || a->W < 1) {
        set_error("%s: nv, H and W must be >= 1 (got nv = %d, %d x %d)", who, a->nv, a->H, a->W);
        return NB_ERR_BAD_ARG;
    }
    if (a->nx < 1 || a->ny < 1 || a->nz < 1) {
        set_error("%s: grid dims must be >= 1 (got %d x %d x %d)", who, a->nx, a->ny, a->nz);
        return NB_ERR_BAD_ARG;
    }
    const long long n = (long long)a->nx * a->ny * a->nz;
    if (n > (1LL << 31)) {
        set_error("%s: a %d x %d x %d grid has more than 2^31 points", who, a->nx, a->ny, a->nz);
        return NB_ERR_UNSUPPORTED;
    }
    InsideGrid<T> g;
    g.x = a->x; g.y = a->y; g.z = a->z;
    g.ny = (unsigned)a->ny; g.nz = (unsigned)a->nz; g.n = (unsigned)n;
    g.msks = a->msks; g.RT = RT; g.Ks = Ks;
    g.nv = a->nv; g.H = a->H; g.W = a->W;
    g.inside = a->inside;
    mesh_inside_kernel<T><<<(unsigned)((n + kInsideThreads - 1) / kInsideThreads), kInsideThreads, 0, (cudaStream_t)stream>>>(g);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // namespace
}  // namespace nb
