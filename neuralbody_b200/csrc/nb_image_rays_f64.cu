// nb_image_rays_f64 (the multi-view demo / perform sets' float64 camera, and the training datasets' test split, whose K may
// be float32): the double instantiations of nb_image_rays.cuh, in
// its own translation unit so that each object holds one instance of the kernels.
#include "nb_image_rays.cuh"

using namespace nb;

extern "C" {

int nb_image_rays_f64(const nb_image_rays_args* a, const double K_inv[9], const double R[9], const double T[3],
                      const double o[3], void* stream) {
    if (a && a->k_f32)      // People-Snapshot's test split: float32 K (K_inv's values are float32's), float64 R and T
        return image_rays_launch<float, double>("nb_image_rays_f64", a, K_inv, R, T, o, stream);
    return image_rays_launch<double, double>("nb_image_rays_f64", a, K_inv, R, T, o, stream);
}

}  // extern "C"
