// nb_image_rays (the People-Snapshot demo's float32 camera) and the workspace size of both entry points:
// the float instantiation of nb_image_rays.cuh.
#include "nb_image_rays.cuh"

using namespace nb;

extern "C" {

size_t nb_image_rays_workspace_bytes(int H, int W) {
    const int n = image_rays_pixels(H, W);
    if (n < 0) return 0;
    const size_t sb = image_rays_scan_bytes(n);
    if (sb == 0) return 0;
    return align256((size_t)n * sizeof(int)) + align256(sb);
}

int nb_image_rays(const nb_image_rays_args* a, const float K_inv[9], const float R[9], const float T[3], const float o[3],
                  void* stream) {
    if (a && a->k_f32) {
        set_error("nb_image_rays: k_f32 is for nb_image_rays_f64 (a float32 K with a float64 R and T)");
        return NB_ERR_BAD_ARG;
    }
    return image_rays_launch<float, float>("nb_image_rays", a, K_inv, R, T, o, stream);
}

}  // extern "C"
