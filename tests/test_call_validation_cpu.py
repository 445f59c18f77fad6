"""CPU: every entry point that takes an nb_render_args validates the frame fields (batch, R, Th, bounds, voxel_size, out_sh,
level_dims, the volume and weight blobs), the render calls also validate the ray fields, and each reports an error under its
own name.  The device pointers here are placeholders: every call in this file is rejected before it makes a CUDA call."""
import ctypes
import subprocess

import pytest

from neuralbody_b200 import capi

NB_ERR_BAD_ARG = -1
FAKE = 0x10000      # placeholder device address, never dereferenced
RAY_FIELDS = ("ray_o", "ray_d", "near", "far", "rgb_map", "disp_map", "acc_map", "depth_map")
ENTRY_POINTS = ("nb_render_fwd", "nb_render_bwd", "nb_decode_density", "nb_decode_density_list")


def _args():
    """A call whose frame and ray fields all pass validation."""
    a = capi.nb_render_args()
    a.batch, a.n_rays, a.n_samples = 1, 4, 8
    for name in ("R", "Th", "bounds", "volume_blob", "weights_blob") + RAY_FIELDS:
        setattr(a, name, FAKE)
    for i in range(3):
        a.voxel_size[i], a.out_sh[i] = 0.005, 64
    for l, c in enumerate((32, 64, 128, 128)):
        a.level_dims[l][0], a.level_dims[l][1], a.level_dims[l][2], a.level_dims[l][3] = c, 16, 16, 16
    a.volume_dtype = capi.NB_DTYPE_F32
    return a


def _call(entry, a):
    lib = capi.load()
    if entry == "nb_render_fwd":
        return lib.nb_render_fwd(ctypes.byref(a), None)
    if entry == "nb_render_bwd":
        b = capi.nb_render_bwd_args()
        b.fwd = ctypes.pointer(a)
        b.save, b.raw, b.workspace, b.workspace_bytes = FAKE, FAKE, FAKE, 1 << 40
        b.weights, b.grads = ctypes.pointer(capi.nb_decoder_weights()), ctypes.pointer(capi.nb_decoder_weights())
        return lib.nb_render_bwd(ctypes.byref(b), None)
    if entry == "nb_decode_density_list":
        a.precision = capi.NB_PRECISION_TC_FP16X3
        a.workspace, a.workspace_bytes = FAKE, 1 << 40
    return getattr(lib, entry)(ctypes.byref(a), FAKE, 16, FAKE, None)


def _error():
    return capi.load().nb_last_error().decode()


FRAME_DEFECTS = {
    "batch": lambda a: setattr(a, "batch", 0),
    "R": lambda a: setattr(a, "R", None),
    "bounds": lambda a: setattr(a, "bounds", None),
    "weights_blob": lambda a: setattr(a, "weights_blob", None),
    "volume_dtype": lambda a: setattr(a, "volume_dtype", 7),
    "level_dims": lambda a: a.level_dims[2].__setitem__(1, 0),
    "voxel_size": lambda a: a.voxel_size.__setitem__(1, 0.0),
}


@pytest.mark.parametrize("entry", ENTRY_POINTS)
@pytest.mark.parametrize("defect", sorted(FRAME_DEFECTS))
def test_frame_field_rejected_under_the_entry_points_name(built_lib, entry, defect):
    a = _args()
    FRAME_DEFECTS[defect](a)
    assert _call(entry, a) == NB_ERR_BAD_ARG
    assert _error().startswith(entry + ":"), _error()


@pytest.mark.parametrize("entry", ("nb_render_fwd", "nb_render_bwd"))
@pytest.mark.parametrize("field", ("ray_o", "far", "depth_map"))
def test_ray_field_rejected_by_the_render_calls(built_lib, entry, field):
    a = _args()
    setattr(a, field, None)
    assert _call(entry, a) == NB_ERR_BAD_ARG
    assert _error().startswith(entry + ":") and "null" in _error(), _error()


@pytest.mark.parametrize("entry", ("nb_decode_density", "nb_decode_density_list"))
def test_density_calls_report_the_frame_error_not_the_missing_rays(built_lib, entry):
    """The density calls read no ray field: with all of them null, the call fails on its frame alone."""
    a = _args()
    a.n_rays = a.n_samples = 0
    for name in RAY_FIELDS:
        setattr(a, name, None)
    a.weights_blob = None
    assert _call(entry, a) == NB_ERR_BAD_ARG
    msg = _error()
    assert msg.startswith(entry + ":") and "weights_blob" in msg and "ray" not in msg, msg


def test_library_exports_no_internal_symbols(built_lib):
    out = subprocess.run(["nm", "-D", "--defined-only", built_lib], capture_output=True, text=True, check=True).stdout
    names = [line.split()[-1] for line in out.splitlines() if line.strip()]
    assert "nb_render_fwd" in names
    assert not [n for n in names if n.startswith("nbi_")]
