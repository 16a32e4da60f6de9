"""Device-side counterpart of the reference's tools/visualization.py (import as device.tools.visualization):
render_animation with the reference's signature, its frames rasterised on the device (gast_b200.render,
DESIGN.md §8.5) and piped to ffmpeg.

As in the reference, each 3D panel's x and y limits follow its pose's root joint (visualization.py:166-167), and the
2D bones are drawn when the skeleton has as many joints as the keypoints and the layout is not COCO.  The root it
follows is that of the drawn, skipped frame (the reference reads its trajectories without input_video_skip).  Only
bones of joints below 17 are drawn.  Differences from the reference: only .mp4 output (a .gif raises GastError;
render the frames with gast_b200.render.render_frames and encode them yourself), ffmpeg must be on PATH (GastError
otherwise), and the picture is the project's rasterisation, not matplotlib's.
"""
import numpy as np

from gast_b200 import render as _R
from gast_b200.render import downsample_frames, read_video  # noqa: F401  (the reference module's helpers)

__all__ = ['render_animation', 'read_video', 'downsample_frames']


def render_animation(keypoints, keypoints_metadata, poses, skeleton, fps, bitrate, azim, output, viewport,
                     limit=-1, downsample=1, size=6, input_video_path=None, input_video_skip=0):
    """visualization.py:84-227: keypoints (T, J, 2) in image pixels, poses a dict of (T, J, 3) world poses, one 3D
    panel each (trainval.py --render: 'Reconstruction' and 'Ground truth')"""
    bones_2d = len(skeleton.parents()) == int(np.shape(keypoints)[1]) and keypoints_metadata['layout_name'] != 'coco'
    _R.render_animation(keypoints, keypoints_metadata, poses, skeleton, fps, bitrate, azim, output, viewport, limit,
                        downsample, size, input_video_path, input_video_skip, follow_root=True, bones_2d=bones_2d)
