"""Config surface of the render hot path.

Mirrors the keys the reference reads inside the path (lib/config/config.py:9-129 +
the yaml-only keys of configs/snapshot_exp/snapshot_f3c.yaml:55-78):
  N_samples, perturb, raw_noise_std, white_bkgd   if_clight_renderer.py:13,16,82
  voxel_size                                      latent_xyzc.py:54
  xyz_res, view_res                               embedder.py:53-54
  num_train_frame                                 latent_xyzc.py:16
  H, W, ratio, N_rand, chunk
  network_module/path, renderer_module/path       make_network.py / make_renderer.py
Same yaml format (`parent_cfg` inheritance, config.py:149-152) and the same trailing
`KEY VALUE` override form (config.py:153).  Unlike upstream nothing is parsed from
sys.argv at import time and open3d is not imported.
"""
import ast
import copy
import os

import yaml

_PKG_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class CfgNode(dict):
    """Attribute-style dict; nested dicts become CfgNodes (a minimal stand-in for yacs)."""

    def __init__(self, init=None):
        super().__init__()
        for k, v in (init or {}).items():
            self[k] = CfgNode(v) if isinstance(v, dict) and not isinstance(v, CfgNode) else v

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name)

    def __setattr__(self, name, value):
        self[name] = CfgNode(value) if isinstance(value, dict) and not isinstance(value, CfgNode) else value

    def clone(self):
        return copy.deepcopy(self)

    def merge_from_other_cfg(self, other):
        for k, v in other.items():
            if isinstance(v, dict) and isinstance(self.get(k), dict):
                self[k].merge_from_other_cfg(v)
            else:
                self[k] = CfgNode(v) if isinstance(v, dict) and not isinstance(v, CfgNode) else copy.deepcopy(v)

    def merge_from_file(self, path):
        with open(path, "r") as f:
            cur = yaml.safe_load(f) or {}
        if "parent_cfg" in cur:
            parent = cur["parent_cfg"]
            if not os.path.isabs(parent) and not os.path.exists(parent):
                parent = os.path.join(os.path.dirname(path), os.path.basename(parent))
            self.merge_from_file(parent)
        self.merge_from_other_cfg(cur)

    def merge_from_list(self, opts):
        opts = list(opts or [])
        if len(opts) % 2:
            raise ValueError("override list must be KEY VALUE pairs, got %r" % (opts,))
        for key, val in zip(opts[0::2], opts[1::2]):
            node = self
            parts = key.split(".")
            for p in parts[:-1]:
                node = node.setdefault(p, CfgNode())
            if isinstance(val, str):
                try:
                    val = ast.literal_eval(val)
                except (ValueError, SyntaxError):
                    pass
            node[parts[-1]] = val


def _defaults():
    c = CfgNode()
    c.task = "if_nerf"
    c.exp_name = "synth_313"
    c.gpus = [0]
    # plugin selection (make_network.py:5-9 / make_renderer.py:5-9)
    c.network_module = "neuralbody_b200.lib.networks.latent_xyzc"
    c.network_path = os.path.join(_PKG_ROOT, "lib/networks/latent_xyzc.py")
    c.renderer_module = "neuralbody_b200.lib.networks.renderer.if_nerf_renderer"
    c.renderer_path = os.path.join(_PKG_ROOT, "lib/networks/renderer/if_nerf_renderer.py")
    # rendering options (snapshot_f3c.yaml:55-66)
    c.xyz_res = 10
    c.view_res = 4
    c.raw_noise_std = 0
    c.N_samples = 64
    c.N_importance = 128
    c.N_rand = 1024
    c.perturb = 1
    c.white_bkgd = False
    c.num_render_views = 50
    # data options (config.py:14-36, latent_xyzc_313.yaml:74-79)
    c.H = 1024
    c.W = 1024
    c.ratio = 0.5
    c.num_train_frame = 60
    c.begin_ith_frame = 0               # the dataset's first frame (config.py:22)
    c.ith_frame = 0                     # the frame the multi-view demo renders from every view (config.py:25)
    c.voxel_size = [0.005, 0.005, 0.005]
    c.big_box = False
    c.mask_bkgd = True                  # the training datasets' background (config.py:31)
    c.body_sample_ratio = 0.5           # sample_ray's class split (config.py:128-129)
    c.face_sample_ratio = 0.
    c.dataset_image_steps = 'host'      # the training datasets' undistort / resize / background: 'host' (upstream's cv2
                                        # steps in the item) | 'device' (the item ships the decoded image and mask;
                                        # nb_item_images runs the steps on the GPU, bit for bit)
    # evaluation (config.py:111, 120 upstream; the evaluator plugin as make_evaluator.py:5-9 selects it)
    c.evaluator_module = "neuralbody_b200.lib.evaluators.if_nerf"
    c.evaluator_path = os.path.join(_PKG_ROOT, "lib/evaluators/if_nerf.py")
    c.result_dir = 'data/result'
    c.eval_whole_img = False
    # the demo modes' visualizer plugin (make_visualizer.py:5-9; novel_view_cfg / rotate_smpl_cfg select if_nerf_demo,
    # novel_pose_cfg if_nerf_perform)
    c.visualizer_module = "neuralbody_b200.lib.visualizers.if_nerf_demo"
    c.visualizer_path = os.path.join(_PKG_ROOT, "lib/visualizers/if_nerf_demo.py")
    c.mesh_th = 50                      # isovalue of the mesh renderer's marching cubes, on raw sigma (config.py:45)
    c.mesh_output = 'host'              # the mesh renderer's outputs: 'host' (upstream's float64 numpy cube and host mesh) |
                                        # 'device' (the fp32 CUDA cube and a mcubes.DeviceMesh, nothing copied back)
    c.sparse_encode = 'reference'       # the SparseConvNet encode: 'reference' (upstream's spconv module) | 'dense' (the
                                        # dense-PyTorch emulation) | 'cuda' (sparse convolutions on the GPU, nb_spconv)
    # H100 renderer options (new)
    c.render_precision = "tc_fp16x3"    # "fp32" exact FFMA kernel | "tc_fp16x3" wgmma, 3-pass hi/lo density path
                                        # (meets the 1e-3 parity gate) | "tc_fp16" wgmma 1-pass (fastest, ~4e-3 on depth)
    c.render_volume_dtype = "auto"      # "auto": fp16 volume for tc_fp16, fp32 otherwise | "fp32" | "fp16".  A training call on
                                        # the exact kernel (render_train_precision 'fp32') packs fp32 whatever this says: its
                                        # backward reads the fp32 volume only
    c.render_skip_empty = True          # tensor-core modes: exact empty-sample skipping (bit-identical outputs)
    c.render_return_weights = True      # 'weights' (B,n,S) is unused downstream; may be skipped
    c.render_train_precision = 'tc_tf32x3'   # calls autograd records: 'tc_tf32x3' (wgmma TF32 GEMM chains over the sample list) | 'fp32' (exact FFMA kernels)
    c.render_importance = 0             # f-4: > 0 adds a fine pass with this many importance samples (upstream's N_importance is a dead key for Neural Body, so the default stays single-pass)
    c.chunk = 0                         # 0 = all rays of the call in one launch
    return c


cfg = _defaults()


def make_cfg(cfg_file=None, opts=None, target=None):
    """Build (in place) a config from defaults + yaml (+ parent_cfg) + KEY VALUE overrides."""
    c = target if target is not None else cfg
    if cfg_file:
        c.merge_from_file(cfg_file)
    c.merge_from_list(opts)
    return c


def get_active_cfg():
    """When running inside the reference process (its `lib.config` already imported, e.g. the
    renderer was selected through the reference's own make_renderer), read the reference's
    singleton so yaml/CLI overrides made there are honoured; otherwise use ours."""
    import sys
    mod = sys.modules.get("lib.config")
    if mod is not None and hasattr(mod, "cfg"):
        return mod.cfg
    return cfg
