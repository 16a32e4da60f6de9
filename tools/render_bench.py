"""GPU: rendering the video demo's animation frames with gast_b200.render.

The clip has the baseball demo's shape (277 frames at 1920 x 1080, 17 joints, one person, one 3D panel) with seeded
synthetic keypoints and poses; panels are S = size * dpi = 500 pixels, so each frame is 500 x 1000 RGB.  Timed, with
and without a synthetic 1920 x 1080 background video:
  * render: one render_frames call over the whole clip (inputs already on the device), CUDA events, `--reps` times
    after a warm-up;
  * to_pipe: render_animation's .mp4 path (chunks rendered, copied to pinned memory and written to a pipe) into an
    `ffmpeg` stand-in that discards its input, host clock, so encoding is not included.
The reference's render_animation (matplotlib + ffmpeg, oracle/_ref/tools/visualization.py) is timed as well when
matplotlib and ffmpeg are both installed; otherwise its line says it was not measured.
Prints one JSON line per measurement, the first with the card's name and power limit read in the same run.

    python tools/render_bench.py [--frames 277] [--size 5] [--reps 5]
"""
import argparse
import json
import os
import shutil
import stat
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, 'gast-net-3dposeestimation_b200')
sys.path[:0] = [PKG, REPO, os.path.dirname(os.path.abspath(__file__))]
from gast_b200 import render as R  # noqa: E402
from eval_bench import card  # noqa: E402

H36M = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]
META = {'keypoints_symmetry': ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]), 'layout_name': 'h36m'}
W, H = 1920, 1080


class Skeleton(object):
    def parents(self):
        return np.array(H36M)

    def joints_right(self):
        return META['keypoints_symmetry'][1]


def clip(T, seed=0):
    rs = np.random.RandomState(seed)
    centre = np.array([W / 2, H / 2]) + 200 * np.sin(np.arange(T)[:, None] / 40. + np.array([0., 1.]))
    kp = (centre[:, None, None, :] + rs.normal(0, 120, (T, 1, 17, 2))).astype(np.float32)
    pose = (np.array([0., 0., 0.9]) + rs.normal(0, 0.35, (T, 17, 3))).astype(np.float32)
    video = rs.randint(0, 256, (T, H, W, 3)).astype(np.uint8)
    return kp, pose, video


def time_render(scene, reps):
    out = scene.render()                                   # warm-up, and the buffer reused below
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        start.record()
        scene.render(out=out)
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return times


def time_to_pipe(scene, reps, tmp):
    times = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        R.write_mp4(scene, os.path.join(tmp, 'o.mp4'), 25, 3000)
        times.append((time.perf_counter() - t0) * 1e3)
    return times[1:]


def reference(kp, pose, video_path, T):
    """the staged reference render_animation, when matplotlib and ffmpeg exist: (ms, reason)"""
    try:
        import matplotlib  # noqa: F401
    except ImportError:
        return None, 'matplotlib is not installed'
    if shutil.which('ffmpeg') is None:
        return None, 'ffmpeg is not on PATH'
    sys.path.insert(0, os.path.join(REPO, 'oracle', '_ref'))
    from tools.visualization import render_animation
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        render_animation(kp[:, 0], META, {'Reconstruction': pose}, Skeleton(), 25, 3000, 70.,
                         os.path.join(d, 'ref.mp4'), (W, H), size=5, input_video_path=video_path)
        return (time.perf_counter() - t0) * 1e3, 'matplotlib + ffmpeg, host clock'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=277)
    ap.add_argument('--size', type=float, default=5)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    kp, pose, video = clip(a.frames)
    first = True
    with tempfile.TemporaryDirectory() as tmp:
        stub = os.path.join(tmp, 'bin', 'ffmpeg')
        os.makedirs(os.path.dirname(stub))
        with open(stub, 'w') as f:
            f.write('#!/bin/sh\ncat > /dev/null\n')
        os.chmod(stub, os.stat(stub).st_mode | stat.S_IXUSR)
        real_path = os.environ.get('PATH', '')
        dkp, dpose, dvid = torch.from_numpy(kp).cuda(), torch.from_numpy(pose).cuda(), torch.from_numpy(video).cuda()
        for bg in ('black', 'video'):
            sc = R.Scene(dkp, {'Reconstruction': dpose}, Skeleton(), 70., (W, H), size=a.size,
                         input_frames=dvid if bg == 'video' else None, keypoints_metadata=META)
            ms = time_render(sc, a.reps)
            os.environ['PATH'] = os.path.dirname(stub) + os.pathsep + real_path
            try:
                pipe = time_to_pipe(sc, max(2, a.reps // 2), tmp)
            finally:
                os.environ['PATH'] = real_path
            row = {'background': bg, 'frames': sc.n_frames, 'frame_shape': list(sc.frame_shape),
                   'render_ms': [round(t, 3) for t in ms],
                   'render_us_per_frame': [round(1e3 * t / sc.n_frames, 2) for t in ms],
                   'to_pipe_ms': [round(t, 1) for t in pipe]}
            if first:
                row['card'] = card()
                first = False
            print(json.dumps(row), flush=True)
        del dvid
    ref_ms, why = None, None
    if shutil.which('ffmpeg') is not None:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, 'clip.mp4')
            import subprocess
            p = subprocess.Popen(['ffmpeg', '-y', '-v', 'error', '-f', 'rawvideo', '-pix_fmt', 'rgb24', '-s', '%dx%d' % (W, H),
                                  '-r', '25', '-i', '-', path], stdin=subprocess.PIPE)
            p.stdin.write(video.tobytes())
            p.stdin.close()
            p.wait()
            ref_ms, why = reference(kp, pose, path, a.frames)
    else:
        why = 'ffmpeg is not on PATH'
    print(json.dumps({'reference_render_animation_ms': ref_ms, 'note': why,
                      'measured': ref_ms is not None}), flush=True)


if __name__ == '__main__':
    main()
