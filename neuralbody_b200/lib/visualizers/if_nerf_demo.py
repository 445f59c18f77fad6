"""Drop-in for the reference's lib/visualizers/if_nerf_demo.py (selected by `visualizer_module` / `visualizer_path`, as
upstream's make_visualizer loads it; `novel_view_cfg` and `rotate_smpl_cfg`): the same `Visualizer()` and
`visualize(output, batch)`, writing data/render/{exp_name}/frame_{frame_index:04d}/{view_index:04d}.png with upstream's
bytes, with the image built on the GPU and written by a background thread (frame_writer.FrameVisualizer; call flush() to
wait for the files)."""
import os

from neuralbody_b200.lib.visualizers.frame_writer import FrameVisualizer


class Visualizer(FrameVisualizer):
    def data_dir(self, exp_name):
        return 'data/render/{}'.format(exp_name)

    def frame_path(self, exp_name, frame_index, view_index):
        return os.path.join('data/render/{}/frame_{:04d}'.format(exp_name, frame_index), '{:04d}.png'.format(view_index))
