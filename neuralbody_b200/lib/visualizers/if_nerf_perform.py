"""Drop-in for the reference's lib/visualizers/if_nerf_perform.py (selected by `visualizer_module` / `visualizer_path`;
`novel_pose_cfg`): as if_nerf_demo's drop-in, writing data/perform/{exp_name}/0/frame{frame_index:04d}_view{view_index:04d}.png."""
import os

from neuralbody_b200.lib.visualizers.frame_writer import FrameVisualizer


class Visualizer(FrameVisualizer):
    def data_dir(self, exp_name):
        return 'data/perform/{}'.format(exp_name)

    def frame_path(self, exp_name, frame_index, view_index):
        return os.path.join('data/perform/{}/{}'.format(exp_name, 0),
                            'frame{:04d}_view{:04d}.png'.format(frame_index, view_index))
