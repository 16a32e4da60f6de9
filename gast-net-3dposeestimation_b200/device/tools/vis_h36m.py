"""Device-side counterpart of the reference's tools/vis_h36m.py (import as device.tools.vis_h36m): render_animation
with the reference's signature, its frames rasterised on the device (gast_b200.render, DESIGN.md §8.5) and piped to
ffmpeg.

Differences from the reference: only .mp4 output (a .gif raises GastError; render the frames with
gast_b200.render.render_frames and encode them yourself), ffmpeg must be on PATH (GastError otherwise), and the
picture is the project's rasterisation, not matplotlib's (no axis panes, grid or ticks).
"""
from gast_b200 import render as _R
from gast_b200.render import downsample_frames, read_video  # noqa: F401  (the reference module's helpers)

__all__ = ['render_animation', 'read_video', 'downsample_frames']


def render_animation(keypoints, keypoints_metadata, poses, skeleton, fps, bitrate, azim, output, viewport, limit=-1,
                     downsample=1, size=5, input_video_path=None, com_reconstrcution=False, input_video_skip=0):
    """vis_h36m.py:58-249: keypoints (T, M, 17, 2) in image pixels, poses a dict of (T, J, 3) world poses, one 3D panel
    each, or one shared panel for two persons with com_reconstrcution"""
    _R.render_animation(keypoints, keypoints_metadata, poses, skeleton, fps, bitrate, azim, output, viewport, limit,
                        downsample, size, input_video_path, input_video_skip, com_reconstrcution=com_reconstrcution)
