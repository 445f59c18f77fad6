"""GPU: nb_mesh_ply against Mesh.export's bytes (the golden frame's mesh, random meshes at word and block edges, special
float64 bits, out-of-range faces with guard bytes), the mesh renderer's `mesh_output: 'device'` against 'host' on the
golden, full-size, multi-view and monocular mask-view frames, and the mesh visualizer drop-in end to end, also under
torch.cuda.set_sync_debug_mode("error")."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

from neuralbody_b200 import capi, mcubes
from test_mesh_ply_cpu import MESH_VISUALIZER, ply_body, random_mesh
from test_mesh_inside_gpu import _case, _mask_batch, _mesh_renderer, _render
from test_mesh_inside_f64_gpu import _batches

pytestmark = pytest.mark.gpu

GUARD = 0xA5


def _export(v, f):
    return mcubes.Mesh(v, f).export(io.BytesIO())


def _device(v, f):
    return mcubes.DeviceMesh(torch.from_numpy(np.ascontiguousarray(v, np.float64)).cuda(),
                             torch.from_numpy(np.ascontiguousarray(f, np.int64)).cuda())


def _pack_with_guard(v, f, guard=64):
    """nb_mesh_ply through the C ABI into a buffer of exactly NB_MESH_PLY_BODY_OFFSET + nb_mesh_ply_bytes bytes followed by
    `guard` guard bytes -> (status, body bytes, guard bytes)."""
    lib = capi.load()
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float64)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f, np.int64)).cuda()
    n = capi.NB_MESH_PLY_BODY_OFFSET + int(lib.nb_mesh_ply_bytes(len(v), len(f)))
    buf = torch.full((n + guard,), GUARD, dtype=torch.uint8, device="cuda")
    a = capi.nb_mesh_ply_args()
    a.nv, a.nf = len(v), len(f)
    a.vertices, a.faces = vt.data_ptr() or None, ft.data_ptr() or None
    a.out, a.out_bytes = buf.data_ptr(), n
    capi.check(lib.nb_mesh_ply(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "nb_mesh_ply")
    host = buf.cpu().numpy()
    status = capi.nb_mesh_ply_result.from_buffer_copy(host[:C.sizeof(capi.nb_mesh_ply_result)].tobytes()).status
    return status, host[capi.NB_MESH_PLY_BODY_OFFSET:n].tobytes(), host[n:]


def _assert_packs_as_export(v, f):
    status, body, guard = _pack_with_guard(v, f)
    assert status == capi.NB_MESH_PLY_OK
    assert body == ply_body(v, f)
    assert (guard == GUARD).all()
    assert _device(v, f).export(io.BytesIO()) == _export(v, f)


# ----------------------------------------------------------------------------- the kernel
SIZES = [0, 1, 31, 32, 33, 100003]


@pytest.mark.parametrize("nv", SIZES)
@pytest.mark.parametrize("nf", SIZES)
def test_random_meshes(nv, nf):
    if nv == 0 and nf > 0:
        f = np.zeros((nf, 3), np.int64)          # Mesh.export's bound is max(V, 1): index 0 of an empty vertex list
        _assert_packs_as_export(np.zeros((0, 3)), f)
        return
    v, f = random_mesh(nv, nf, 1000 * nv + nf)
    _assert_packs_as_export(v, f)


def test_faces_at_both_ends_and_special_vertex_bits():
    v = np.array([[-0.0, np.nan, np.inf], [-np.inf, 5e-324, -2.2250738585072014e-308], [1e308, -1e-310, 0.0]])
    nan_payload = np.array([0x7FF8DEADBEEF0001, -0x0007_0000_0000_0001], np.int64).view(np.float64)
    v = np.concatenate([v, np.stack([nan_payload, nan_payload[::-1], [0.0, -0.0]], axis=1), np.random.RandomState(3).randn(29, 3)])
    V = len(v)
    f = np.array([[0, V - 1, 0], [V - 1, V - 1, V - 1], [0, 0, 0], [1, V - 2, 2]] * 9, np.int64)
    _assert_packs_as_export(v, f)
    status, body, _ = _pack_with_guard(v, f)
    assert np.frombuffer(body[:24 * V], "<i8").tobytes() == v.tobytes()      # the exact bits, NaN payloads included


def test_golden_frame_mesh():
    """The mesh of the golden frame (mesh_s03) as the renderer's host mode returns it."""
    scene, masks, batch = _case("mesh_s03")
    out = _render(_mesh_renderer(scene), batch, "fp32")
    v, f = np.asarray(out["mesh"].vertices), np.asarray(out["mesh"].faces)
    assert len(f) > 1000
    _assert_packs_as_export(v, f)


@pytest.mark.parametrize("bad", [-1, "V"])
def test_out_of_range_faces(bad, tmp_path):
    for nv, nf, at in ((33, 100, 0), (1000, 100003, 100002), (5, 1, 0)):
        v, f = random_mesh(nv, nf, nv)
        f[at, at % 3] = -1 if bad == -1 else nv
        status, body, guard = _pack_with_guard(v, f)
        assert status == capi.NB_MESH_PLY_FACE and (guard == GUARD).all()
        with pytest.raises(ValueError, match="face indices out of range") as want:
            mcubes.Mesh(v, f).export(io.BytesIO())
        p = tmp_path / "bad.ply"
        with pytest.raises(ValueError, match=str(want.value)):
            _device(v, f).export(str(p))
        assert not p.exists()
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------- the renderer's mesh_output
def _render_as(ren, batch, precision, mode, mesh_th=10.0):
    from neuralbody_b200.lib.config import cfg
    old = cfg.mesh_output
    cfg.mesh_output = mode
    try:
        return _render(ren, batch, precision, mesh_th)
    finally:
        cfg.mesh_output = old


def _assert_device_equals_host(ren, batch, precision):
    host = _render_as(ren, batch, precision, "host")
    dev = _render_as(ren, batch, precision, "device")
    cube, mesh = dev["cube"], dev["mesh"]
    assert isinstance(mesh, mcubes.DeviceMesh) and mesh.vertices.is_cuda and mesh.faces.is_cuda
    assert cube.is_cuda and cube.dtype == torch.float32 and tuple(cube.shape) == host["cube"].shape
    np.testing.assert_array_equal(cube.double().cpu().numpy().view(np.int64), host["cube"].view(np.int64))
    hv, hf = np.asarray(host["mesh"].vertices), np.asarray(host["mesh"].faces)
    assert (mesh.nv, mesh.nf) == (len(hv), len(hf)) and len(hf) > 1000
    np.testing.assert_array_equal(mesh.vertices.cpu().numpy().view(np.int64), hv.view(np.int64))
    np.testing.assert_array_equal(mesh.faces.cpu().numpy(), hf)
    assert mesh.export(io.BytesIO()) == _export(hv, hf)
    return host, dev


@pytest.mark.parametrize("name", ["mesh_s03", "mesh_full"])
def test_device_output_equals_host_output(name):
    scene, masks, batch = _case(name)
    ren = _mesh_renderer(scene)
    _assert_device_equals_host(ren, batch, "tc_fp16x3")
    if name == "mesh_s03":
        _assert_device_equals_host(ren, batch, "fp32")
        _assert_device_equals_host(ren, _mask_batch(batch, scene, masks), "fp32")    # float32 multi-view mask views


def test_device_output_equals_host_output_monocular():
    scene, _, masks = _batches("mono_s03")                                          # float64 monocular mask view
    assert masks["RT"].dtype == torch.float64
    _assert_device_equals_host(_mesh_renderer(scene), masks, "tc_fp16x3")


# ----------------------------------------------------------------------------- the visualizer
def _visualizer(monkeypatch, tmp_path):
    from neuralbody_b200.lib.config import get_active_cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    monkeypatch.chdir(tmp_path)
    monkeypatch.setitem(get_active_cfg(), "result_dir", "res")
    return load_source("neuralbody_b200.lib.visualizers.if_nerf_mesh", MESH_VISUALIZER).Visualizer()


def test_render_and_visualize_end_to_end(monkeypatch, tmp_path):
    """Frames at different isovalues through render('device') and the drop-in, then flush(): each file is Mesh.export's bytes
    of the host-mode mesh and reads back; the host-mode meshes through the drop-in write the same files."""
    scene, masks, batch = _case("mesh_s03")
    ren = _mesh_renderer(scene)
    vis = _visualizer(monkeypatch, tmp_path)
    frames = [(3, 10.0), (4, 15.0), (17, 5.0), (5, 10.0), (6, 12.0), (7, 8.0)]   # more frames than slots
    want = {}
    for fi, th in frames:
        host = _render_as(ren, batch, "fp32", "host", th)
        want[fi] = (np.asarray(host["mesh"].vertices), np.asarray(host["mesh"].faces))
        out = _render_as(ren, batch, "fp32", "device", th)
        vis.visualize(out, {"frame_index": torch.tensor([fi], device="cuda")})
    vis.flush()
    d = tmp_path / "res" / "mesh"
    assert sorted(os.listdir(d)) == ["%04d.ply" % fi for fi, _ in sorted(frames)]
    for fi, (v, f) in want.items():
        p = d / ("%04d.ply" % fi)
        assert p.read_bytes() == _export(v, f), fi
        rv, rf = mcubes.read_ply(str(p))
        assert np.array_equal(rv.view(np.int64), v.view(np.int64)) and np.array_equal(rf, f)
    dev_files = {fi: (d / ("%04d.ply" % fi)).read_bytes() for fi in want}
    for fi, (v, f) in want.items():
        os.remove(d / ("%04d.ply" % fi))
        vis.visualize({"mesh": mcubes.Mesh(v, f)}, {"frame_index": torch.tensor([fi])})
    vis.flush()
    for fi in want:
        assert (d / ("%04d.ply" % fi)).read_bytes() == dev_files[fi], fi


def test_face_error_is_raised_by_the_next_call(monkeypatch, tmp_path):
    vis = _visualizer(monkeypatch, tmp_path)
    v, f = random_mesh(40, 50, 2)
    bad = f.copy()
    bad[7, 1] = 40
    vis.visualize({"mesh": _device(v, bad)}, {"frame_index": torch.tensor([1], device="cuda")})
    torch.cuda.synchronize()
    vis._writer._q.join()
    with pytest.raises(ValueError, match="face indices out of range"):
        vis.visualize({"mesh": _device(v, f)}, {"frame_index": torch.tensor([2], device="cuda")})
    vis.visualize({"mesh": _device(v, f)}, {"frame_index": torch.tensor([3], device="cuda")})
    vis.flush()
    assert sorted(os.listdir(tmp_path / "res" / "mesh")) == ["0003.ply"]


def test_visualize_does_not_synchronise(monkeypatch, tmp_path):
    scene, masks, batch = _case("mesh_s03")
    ren = _mesh_renderer(scene)
    vis = _visualizer(monkeypatch, tmp_path)
    outs = [_render_as(ren, batch, "fp32", "device", th) for th in (10.0, 9.0, 11.0, 10.0)]
    fi = torch.tensor([9], device="cuda")
    for k, o in enumerate(outs):                             # warm-up: every slot's pinned buffer and event
        vis.visualize(o, {"frame_index": fi + k})
    vis.flush()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for k, o in enumerate(outs):
            vis.visualize(o, {"frame_index": fi + k})
    finally:
        torch.cuda.set_sync_debug_mode(0)
    vis.flush()
    for k, o in enumerate(outs):
        assert (tmp_path / "res" / "mesh" / ("%04d.ply" % (9 + k))).read_bytes() == o["mesh"].cpu().export(io.BytesIO())
