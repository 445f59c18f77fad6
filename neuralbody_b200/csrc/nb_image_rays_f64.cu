// nb_image_rays_f64 (the multi-view demo / perform sets' float64 camera): the double instantiation of nb_image_rays.cuh, in
// its own translation unit so that each object holds one instance of the kernels.
#include "nb_image_rays.cuh"

using namespace nb;

extern "C" {

int nb_image_rays_f64(const nb_image_rays_args* a, const double K_inv[9], const double R[9], const double T[3],
                      const double o[3], void* stream) {
    return image_rays_launch<double>("nb_image_rays_f64", a, K_inv, R, T, o, stream);
}

}  // extern "C"
