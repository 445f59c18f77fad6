// nb_mesh_inside_f64 (the monocular mesh dataset's prepare_inside_pts, float64 camera): mesh_inside_kernel<double> of
// nb_mesh_inside.cuh.  It has its own translation unit so that nb_mcubes.cu keeps exactly the float instantiation.
#include "nb_mesh_inside.cuh"

using namespace nb;

extern "C" {

int nb_mesh_inside_f64(const nb_mesh_inside_args* a, const double* RT, const double* Ks, void* stream) {
    if (!a || !a->x || !a->y || !a->z || !a->msks || !RT || !Ks || !a->inside) {
        set_error("nb_mesh_inside_f64: null argument");
        return NB_ERR_BAD_ARG;
    }
    if (a->RT || a->Ks) {
        set_error("nb_mesh_inside_f64: a->RT and a->Ks must be NULL (the float64 camera is passed as RT and Ks)");
        return NB_ERR_BAD_ARG;
    }
    return mesh_inside_launch<double>("nb_mesh_inside_f64", a, RT, Ks, stream);
}

}  // extern "C"
