"""nb_train_rays: the training datasets' sampler (sample_ray_h36m / sample_ray, split 'train') on the GPU, bit for bit from
upstream's replayed draws, and its Philox mode."""
import numpy as np
import pytest
import torch

from tools import train_rays_case as TC

pytestmark = pytest.mark.gpu

OUT = ("rgb", "ray_o", "ray_d", "near", "far")


def _cam(it):
    from neuralbody_b200 import rays
    return rays.train_camera(it["K"], it["R"], it["T"], it["bounds"])


def _run(items, case, draws="replay", **kw):
    from neuralbody_b200 import rays
    dev = torch.device("cuda:0")
    kinds, cams = zip(*[_cam(it) for it in items])
    img = torch.from_numpy(np.stack([it["img"] for it in items])).to(dev)
    cmap = torch.from_numpy(np.stack([it["class_map"] for it in items])).to(dev)
    d = [it["draws"] for it in items] if draws == "replay" else draws
    return rays.train_rays(img, cmap, np.stack(cams), kinds[0], case[1], case[2], case[3], draws=d, want_coord=True, **kw)


def _same(got, want, label):
    g, w = got.cpu().numpy(), np.asarray(want)
    assert g.shape == w.shape and np.array_equal(g.view(np.uint32), w.astype(np.float32).view(np.uint32)), \
        "%s: %d values differ" % (label, int((g != w).sum()))


@pytest.mark.parametrize("golden", [TC.GOLDEN_MV, TC.GOLDEN_MONO], ids=["multi_view", "monocular"])
def test_replay_reproduces_the_goldens(golden):
    g = TC.load_golden(golden)
    for c, (case, it) in enumerate(zip(g["cases"], g["items"])):
        res = _run([it], case).check()
        for k in OUT:
            _same(getattr(res, k)[0], it[k], "case %d %s" % (c, k))
        W = it["img"].shape[1]
        assert np.array_equal(res.coord[0].cpu().numpy(), it["coord"][:, 0] * W + it["coord"][:, 1])
        assert int(res.rounds[0]) == int(it["rounds"])


@pytest.mark.parametrize("golden", [TC.GOLDEN_MV, TC.GOLDEN_MONO], ids=["multi_view", "monocular"])
def test_replay_batch_of_two(golden):
    """Two different items of one batch (other view or other mask, same N_rand and ratios) each give their own golden, in
    either order."""
    g = TC.load_golden(golden)
    by = {}
    for case, it in zip(g["cases"], g["items"]):
        by.setdefault(case[1:4], []).append(it)
    pairs = [v[:2] for v in by.values() if len(v) >= 2]
    assert pairs, "the golden has no two cases with the same N_rand and ratios"
    key = [k for k, v in by.items() if len(v) >= 2][0]
    for its in (pairs[0], pairs[0][::-1]):
        assert not np.array_equal(its[0]["class_map"], its[1]["class_map"]) or not np.array_equal(its[0]["img"], its[1]["img"])
        res = _run(its, (0,) + key).check()
        for b in range(2):
            for k in OUT:
                _same(getattr(res, k)[b], its[b][k], "item %d %s" % (b, k))


def _restated(it, coord):
    """The restatement's ray_d, near, far and rgb at the row-major pixels `coord` of item `it`."""
    W = it["img"].shape[1]
    K_inv, o = np.linalg.inv(it["K"]), -np.dot(it["R"].T, it["T"]).ravel()
    d = TC.camera_rays_numpy(K_inv, it["R"], it["T"], o, coord // W, coord % W)
    near, far, norm = TC.near_far64(o, d, it["bounds"])
    return d, near, far, norm


def test_philox_batch_of_two_keeps_items_apart():
    """Philox over two different items (other view, camera, box and image) in one batch: each slot lies in its own item's
    classes and carries its own item's ray and colour."""
    g = TC.load_golden(TC.GOLDEN_MV)
    its = [g["items"][0], g["items"][4]]
    assert not np.array_equal(its[0]["K"], its[1]["K"]) or not np.array_equal(its[0]["R"], its[1]["R"])
    torch.manual_seed(2)
    res = _run(its, (0, 3000, 0.5, 0.2), draws=None).check()
    for b, it in enumerate(its):
        coord = res.coord[b].cpu().numpy()
        cm = it["class_map"].reshape(-1)
        assert cm[coord].all()
        d, near, far, norm = _restated(it, coord)
        assert (near < far).all()
        _same(res.ray_d[b], d.astype(np.float32), "item %d ray_d" % b)
        _same(res.near[b], (near / norm).astype(np.float32), "item %d near" % b)
        _same(res.far[b], (far / norm).astype(np.float32), "item %d far" % b)
        _same(res.rgb[b], it["img"].reshape(-1, 3)[coord], "item %d rgb" % b)


@pytest.mark.parametrize("golden", [TC.GOLDEN_MV, TC.GOLDEN_MONO], ids=["multi_view", "monocular"])
def test_test_split_reproduces_the_golden(golden):
    """Split 'test' (the evaluation view): every box-hit ray of the view and its colour, bit for bit upstream's, from the
    camera and the image (nb_image_rays_f64; the monocular golden has a float32 K with float64 R and T)."""
    from neuralbody_b200 import rays
    t = TC.load_golden(golden)["test"]
    kind, cam = rays.train_camera(t["K"], t["R"], t["T"], t["bounds"])
    H, W = t["img"].shape[:2]
    out = rays.dataset_image_rays(cam, kind, H, W, torch.from_numpy(t["img"]).cuda())
    torch.cuda.synchronize()
    for k, got in zip(("ray_o", "ray_d", "near", "far"), out[:4]):
        _same(got, t[k], k)
    assert np.array_equal(out[4].cpu().numpy(), t["mask_at_box"])
    _same(out[5], t["rgb"], "rgb")


def _philox_case(seed, n_rays=3000, rb=0.5, rf=0.2):
    g = TC.load_golden(TC.GOLDEN_MONO)
    it = g["items"][1]           # the mask with label-13 pixels
    torch.manual_seed(seed)
    return it, _run([it], (0, n_rays, rb, rf), draws=None)


def test_philox_slots_lie_in_their_class_and_rays_match_the_restatement():
    it, res = _philox_case(0)
    res.check()
    coord = res.coord[0].cpu().numpy()
    cm = it["class_map"].reshape(-1)
    assert (cm[coord] & (TC.train_item.BODY | TC.train_item.FACE | TC.train_item.BOUND)).all()
    # the rays of the drawn pixels are the restatement's rays of those pixels
    W = it["img"].shape[1]
    K_inv, o = np.linalg.inv(it["K"]), -np.dot(it["R"].T, it["T"]).ravel()
    d = TC.camera_rays_numpy(K_inv, it["R"], it["T"], o, coord // W, coord % W)
    near, far, norm = TC.near_far64(o, d, it["bounds"])
    assert (near < far).all()
    _same(res.ray_d[0], d.astype(np.float32), "ray_d")
    _same(res.near[0], (near / norm).astype(np.float32), "near")
    _same(res.rgb[0], it["img"].reshape(-1, 3)[coord], "rgb")


def test_philox_per_round_split_is_exact_when_nothing_misses():
    """A map whose every class pixel's ray hits the box: one round, n_body body slots, then n_face face, then the rest."""
    it, _ = _philox_case(0)
    hit = dict(it)
    cm = it["class_map"].copy()
    keep = np.zeros_like(cm)
    keep.reshape(-1)[_philox_case(1)[1].coord[0].cpu().numpy()] = 1      # pixels known to hit the box
    hit["class_map"] = np.where(keep == 1, cm, 0).astype(np.uint8)
    torch.manual_seed(3)
    res = _run([hit], (0, 1000, 0.5, 0.2), draws=None).check()
    assert int(res.rounds[0]) == 1
    c = res.coord[0].cpu().numpy()
    m = hit["class_map"].reshape(-1)
    assert (m[c[:500]] & 1).all() and (m[c[500:700]] & 2).all() and (m[c[700:]] & 4).all()


def test_philox_uniform_chi_square():
    """Every bound draw of a small all-hit map: per-pixel counts are uniform (chi-square at a fixed seed)."""
    from scipy import stats
    it, res0 = _philox_case(1)
    pix = np.unique(res0.coord[0].cpu().numpy())[:40]
    cm = np.zeros_like(it["class_map"])
    cm.reshape(-1)[pix] = TC.train_item.BOUND | TC.train_item.BODY
    m = dict(it, class_map=cm)
    torch.manual_seed(11)
    res = _run([m], (0, 40000, 0.0, 0.0), draws=None).check()
    counts = np.bincount(np.searchsorted(pix, res.coord[0].cpu().numpy()), minlength=len(pix))
    p = stats.chisquare(counts).pvalue
    assert p > 1e-3, p


def test_philox_seeding_and_the_cuda_generator():
    a, b, c = _philox_case(5)[1], _philox_case(5)[1], _philox_case(6)[1]
    for r in (a, b, c):
        r.check()
    assert torch.equal(a.ray_d, b.ray_d) and torch.equal(a.rgb, b.rgb)
    assert not torch.equal(a.ray_d, c.ray_d)
    # the key comes from the CPU generator: the CUDA generator, which the jitter's t_rand stream is drawn from, is untouched
    g = TC.load_golden(TC.GOLDEN_MONO)
    state = torch.cuda.get_rng_state()
    _run([g["items"][1]], (0, 3000, 0.5, 0.2), draws=None).check()
    assert torch.equal(torch.cuda.get_rng_state(), state)


def test_sampler_call_does_not_synchronise():
    g = TC.load_golden(TC.GOLDEN_MV)
    it = g["items"][0]
    from neuralbody_b200 import rays
    case = g["cases"][0]
    _run([it], case, draws=None).check()        # warm: library loaded, workspace size queried
    kind, cam = _cam(it)
    img = torch.from_numpy(it["img"][None].copy()).cuda()
    cmap = torch.from_numpy(it["class_map"][None].copy()).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = rays.train_rays(img, cmap, cam[None], kind, case[1], case[2], case[3])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res.check()


def test_all_bound_pixels_missing_raises():
    """A view whose class-map pixels all have rays that miss the box: upstream loops forever, the call reports it."""
    g = TC.load_golden(TC.GOLDEN_MV)
    it = dict(g["items"][0])
    it["bounds"] = (it["bounds"] + np.float32(100.)).astype(np.float32)    # the box far behind the camera's view
    res = _run([it], (0, 1000, 0.5, 0.0), draws=None)
    with pytest.raises(RuntimeError, match="sampling rounds"):
        res.check()


def test_render_step_from_the_image_equals_the_step_from_the_rays():
    """A training step through Renderer.render on the image batch (replayed draws) equals the step on the restatement's
    rays (which equal upstream's, test_train_rays_cpu): the outputs and the loss bit for bit, and the parameter gradients
    to the run-to-run spread of the backward's atomic accumulation (two steps on the same rays differ by as much)."""
    from neuralbody_b200.lib.config import cfg
    from gpu_utils import make_net_and_renderer, BATCH_KEYS
    from tools import mesh_mono_case as MM
    from neuralbody_b200.lib.datasets import train_item
    from neuralbody_b200 import rays
    scene = MM.make_scene(0.3)
    H, W = 100, 75
    K = MM.get_camera(MM.camera_pkl(scene, H, W))["K"].astype(np.float32)
    msk = (MM.silhouette(scene, K.astype(np.float64), H, W, 2) != 0).astype(np.uint8)
    R, T = np.eye(3), np.zeros((3, 1))
    cb = scene["can_bounds"][0].numpy().astype(np.float32)
    ys, xs = np.nonzero(msk)
    bound = np.zeros_like(msk)
    bound[max(ys.min() - 6, 0):ys.max() + 7, max(xs.min() - 6, 0):xs.max() + 7] = 1
    cmap = train_item.class_map_snapshot(msk, bound)
    rng = np.random.RandomState(0)
    img = rng.rand(H, W, 3).astype(np.float32)
    n_rays = 1024
    rgb, ray_o, ray_d, near, far, _, rounds, draws = TC.sample_numpy(img, cmap, K, R, T, cb, n_rays, 0.5, 0.0, None, rng=rng)

    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_train_precision = "tc_tf32x3"
    dev = torch.device("cuda:0")
    outs = []
    for from_image in (False, True):
        net, ren = make_net_and_renderer(scene)
        net.train(True)
        batch = {k: scene[k].to(dev) for k in BATCH_KEYS if k not in ("ray_o", "ray_d", "near", "far")}
        if from_image:
            kind, cam = rays.train_camera(K, R, T, cb)
            batch.update({"img": torch.from_numpy(img)[None].to(dev), "ray_class": torch.from_numpy(cmap)[None].to(dev),
                          "meta": {"train_cam": torch.from_numpy(cam)[None], "train_k_kind": torch.tensor([kind]),
                                   "N_rand": torch.tensor([n_rays]), "body_sample_ratio": torch.tensor([0.5], dtype=torch.float64),
                                   "face_sample_ratio": torch.tensor([0.0], dtype=torch.float64)}})
            ren.train_rays(batch, draws=[draws])
        else:
            batch.update({k: torch.from_numpy(v)[None].to(dev) for k, v in (("ray_o", ray_o), ("ray_d", ray_d), ("near", near),
                                                                              ("far", far), ("rgb", rgb))})
            batch["mask_at_box"] = torch.ones((1, n_rays), dtype=torch.bool, device=dev)
        torch.manual_seed(7)
        ret = ren.render(batch)
        mask = batch["mask_at_box"]
        loss = torch.mean((ret["rgb_map"][mask] - batch["rgb"][mask]) ** 2)
        loss.backward()
        torch.cuda.synchronize()
        outs.append(({k: v.detach().cpu() for k, v in ret.items()}, loss.item(),
                     [p.grad.detach().cpu().clone() for p in net.parameters() if p.grad is not None]))
    (o0, l0, g0), (o1, l1, g1) = outs
    same = lambda a, b: a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))   # NaN disp_map too
    assert l0 == l1
    for k in o0:
        assert same(o0[k], o1[k]), k
    assert len(g0) == len(g1) > 0
    for a, b in zip(g0, g1):
        assert a.shape == b.shape and float((a - b).norm()) <= 1e-5 * float(a.norm()) + 1e-12
