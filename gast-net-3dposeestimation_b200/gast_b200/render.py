"""The reconstruction's animation frames on the device (tools/vis_h36m.py:58-249, tools/visualization.py:84-227).

`render_frames` turns 2D keypoints, lifted 3D poses and optionally the decoded input video into uint8 RGB frames
(F, S, S*(1+P), 3) on the device: the input panel (the video frame fitted into S x S, the 2D bones in pink, the joint
discs black or red with a white edge) and P 3D panels (the skeletons under the reference's view, bones coloured by
`h36m_color_edge`, the nearest bone in front).  The kernel is csrc/render.cuh; its formulas are in DESIGN.md §8.5.
Matplotlib's look (axis panes, grid, ticks, its exact line rasterisation) is not reproduced.

The video's frame selection follows the reference: `input_video_skip` and `limit` as read_video and render_animation
apply them (vis_h36m.py:128-155), `downsample` as downsample_tensor (:53-55), all on the device.  Numpy inputs are
uploaded with one asynchronous copy each; nothing waits for the device.
"""
import ctypes as C
import shutil
import subprocess

import numpy as np
import torch

from . import _lib as L
from .engine import GastError, _check, _p, _stream

ELEV = 15.0             # view_init(elev=15.)
RADIUS = 1.7            # the axis limits' radius
DIST = 7.5              # ax.dist
SHARED_PANEL, FOLLOW_ROOT, BONES_2D = 1, 2, 4       # gast_render_frames flags
MAX_BONE = 17           # index = np.arange(17) (vis_h36m.py:158): bones of joints >= 17 are not drawn

# tools/color_edge.py:12-30 h36m_color_edge, with the RGB values of its comments; every other joint is purple
_COLOR_GROUPS = [([5, 15], (205, 133, 63)),         # peru
                 ([2, 12], (205, 92, 92)),          # indianred
                 ([6, 16], (255, 127, 80)),         # coral
                 ([3, 13], (165, 42, 42)),          # brown
                 ([1, 4, 11, 14], (210, 180, 140)), # tan
                 ([7, 9], (128, 128, 0))]           # olive
_PURPLE = (128, 0, 128)


def color_table(J):
    """(J, 3) uint8: the RGB colour of the bone that ends at each joint (h36m_color_edge)"""
    t = np.empty((J, 3), dtype=np.uint8)
    for j in range(J):
        t[j] = next((c for js, c in _COLOR_GROUPS if j in js), _PURPLE)
    return t


def panel_side(size, dpi):
    """S: a panel's side in pixels, size inches at dpi dots per inch"""
    S = int(round(float(size) * float(dpi)))
    if not 8 <= S <= 8192:
        raise GastError('render: a panel of %r inches at %r dpi is %d pixels (8 .. 8192)' % (size, dpi, S))
    return S


def geometry(S, dpi, Hin, Win, azim, shared=False, elev=ELEV, radius=RADIUS, dist=DIST):
    """the library's float32 geometry of a call (gast_render_geometry): the 3D rows, the image fit, the coverage
    edges and S/2 -- what tests/renderref.py restates the kernel with"""
    geo = (C.c_float * 20)()
    _check(L.load().gast_render_geometry(int(S), float(dpi), int(Hin), int(Win), float(elev), float(azim), float(radius),
                                         float(dist), 1 if shared else 0, geo), 'gast_render_geometry')
    return np.array(geo[:], dtype=np.float32)


def _device(dev):
    if dev is None:
        return torch.device('cuda', torch.cuda.current_device())
    return dev


def _on_device(x, dtype, dev, what):
    """x as a contiguous CUDA tensor of dtype on dev: CUDA tensors are converted on the device, numpy arrays uploaded
    with one asynchronous copy; a CPU tensor is refused (there is no CPU path)"""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise GastError('render: %s must be a CUDA tensor or a numpy array -- there is no CPU path' % what)
        return x.to(device=dev, dtype=dtype).contiguous()
    a = np.ascontiguousarray(np.asarray(x), dtype=torch.empty(0, dtype=dtype).numpy().dtype)
    out = torch.empty(a.shape, dtype=dtype, device=dev)
    if a.size:
        out.copy_(torch.from_numpy(a), non_blocking=True)
    return out


def downsample_frames(x, factor):
    """downsample_tensor (vis_h36m.py:53-55) of a CUDA float32 or uint8 tensor along its first axis, on the device:
    the mean of each group of `factor` frames, numpy's float32 arithmetic (uint8: its float64 mean, truncated)"""
    factor = int(factor)
    if factor < 1:
        raise GastError('render: downsample factor %d < 1' % factor)
    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype not in (torch.float32, torch.uint8):
        raise GastError('render: downsample_frames takes a CUDA float32 or uint8 tensor')
    if factor == 1:
        return x
    x = x.contiguous()
    n = int(x.shape[0]) // factor
    out = torch.empty((n,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    row = 1
    for s in x.shape[1:]:
        row *= int(s)
    if n and row:
        with torch.cuda.device(x.device):
            _check(L.load().gast_downsample_frames(_p(x), int(x.shape[0]), row, factor, 0 if x.dtype == torch.float32 else 1,
                                                   _p(out), C.c_void_p(_stream(x.device))), 'gast_downsample_frames')
    return out


class Scene(object):
    """The inputs of an animation, selected, downsampled and on the device, ready to render any range of its
    `n_frames` frames.  `render_frames` builds one per call; `render_animation` builds one and renders it in chunks."""

    def __init__(self, keypoints, poses, skeleton, azim, viewport, size=5, dpi=100, input_frames=None,
                 com_reconstrcution=False, limit=-1, downsample=1, input_video_skip=0, keypoints_metadata=None,
                 follow_root=False, bones_2d=None, device=None):
        pose_list = list(poses.values()) if isinstance(poses, dict) else list(poses)
        if not pose_list:
            raise GastError('render: at least one 3D pose sequence is required')
        for x, what in [(keypoints, 'keypoints'), (input_frames, 'input_frames')] + [(q, 'poses') for q in pose_list]:
            if isinstance(x, torch.Tensor) and not x.is_cuda:
                raise GastError('render: %s must be a CUDA tensor or a numpy array -- there is no CPU path' % what)
        kshape = tuple(np.shape(keypoints))
        if len(kshape) == 3:
            kshape = kshape[:1] + (1,) + kshape[1:]        # visualization.py's (T, J, 2): one person
        if len(kshape) != 4 or kshape[-1] != 2:
            raise GastError('render: keypoints (T, M, J, 2) or (T, J, 2) expected, got %s' % (tuple(np.shape(keypoints)),))
        M, J = int(kshape[1]), int(kshape[2])
        for q in pose_list:
            if len(np.shape(q)) != 3 or tuple(np.shape(q)[1:]) != (J, 3):
                raise GastError('render: poses (T, %d, 3) expected, got %s' % (J, tuple(np.shape(q))))
        parents = np.asarray(skeleton.parents(), dtype=np.int64)
        if parents.shape != (J,):
            raise GastError('render: the skeleton has %d joints, the keypoints %d' % (parents.size, J))
        if not np.all((parents >= -1) & (parents < J)):
            raise GastError('render: the skeleton\'s parents are not -1 or joints')
        if J > 32 or M * J > 256:
            raise GastError('render: %d persons x %d joints (J <= 32, M*J <= 256)' % (M, J))
        if keypoints_metadata is not None:
            right = list(keypoints_metadata['keypoints_symmetry'][1])
            coco = keypoints_metadata.get('layout_name') == 'coco'
        else:
            right, coco = list(skeleton.joints_right()), False
        if any(not 0 <= int(j) < J for j in right):
            raise GastError('render: right joints %s outside the %d keypoints' % (right, J))
        factor, limit, skip = int(downsample), int(limit), int(input_video_skip)
        if factor < 1 or skip < 0:
            raise GastError('render: downsample must be >= 1 and input_video_skip >= 0')
        shared = bool(com_reconstrcution) and M == 2
        if shared and follow_root:
            raise GastError('render: a shared panel cannot follow one pose\'s root')
        if (not shared and len(pose_list) > 8) or (shared and len(pose_list) * J > 256):
            raise GastError('render: %d pose sequences (at most 8 panels, 256 joints in a shared panel)' % len(pose_list))
        if input_frames is not None:
            vshape = tuple(np.shape(input_frames))
            if len(vshape) != 4 or vshape[-1] != 3 or (isinstance(input_frames, torch.Tensor) and
                                                       input_frames.dtype != torch.uint8):
                raise GastError('render: input_frames (T, H, W, 3) uint8 expected, got %s' % (vshape,))
            Hin, Win = int(vshape[1]), int(vshape[2])
        else:
            Win, Hin = int(viewport[0]), int(viewport[1])
        if Win <= 0 or Hin <= 0:
            raise GastError('render: an input image of %d x %d pixels' % (Win, Hin))
        self.S = panel_side(size, dpi)
        if not float(dpi) > 0:
            raise GastError('render: dpi must be positive')

        if isinstance(keypoints, torch.Tensor) and device is None:
            device = keypoints.device
        dev = _device(device)
        self.device = dev
        kp = _on_device(keypoints, torch.float32, dev, 'keypoints').reshape(kshape)
        ps = [_on_device(q, torch.float32, dev, 'poses') for q in pose_list]
        # frame selection (vis_h36m.py:121-155): the video's frames read_video keeps, the keypoints and poses from
        # the skip on, all cut to the shortest; without a video a black image and no skip
        vid = None
        if input_frames is not None:
            vid = _on_device(input_frames, torch.uint8, dev, 'input_frames')
            vid = vid[skip:] if limit == -1 else vid[skip:max(limit, skip)]
            kp = kp[skip:]
            ps = [q[skip:] for q in ps]
        n = min([int(kp.shape[0])] + [int(q.shape[0]) for q in ps] + ([int(vid.shape[0])] if vid is not None else []))
        kp, ps = kp[:n], [q[:n] for q in ps]
        vid = vid[:n] if vid is not None else None
        if factor > 1:
            kp = downsample_frames(kp, factor)
            ps = [downsample_frames(q, factor) for q in ps]
            vid = downsample_frames(vid, factor) if vid is not None else None
        n //= factor
        self.n_frames = n if limit < 1 else min(limit, n)

        self.dpi, self.azim = float(dpi), float(azim)
        self.keypoints = kp.contiguous()
        self.poses = torch.stack(ps, 0).contiguous()
        self.video = vid.contiguous() if vid is not None else None
        self.Hin, self.Win, self.M, self.J = Hin, Win, M, J
        self.panels = 1 if shared else len(ps)
        if bones_2d is None:                           # vis_h36m.py:184: 17 joints, not the COCO layout
            bones_2d = J == MAX_BONE and not coco
        self.flags = (SHARED_PANEL if shared else 0) | (FOLLOW_ROOT if follow_root else 0) | (BONES_2D if bones_2d else 0)
        self.n_bones = min(J, MAX_BONE)
        self._parents = (C.c_int32 * J)(*[int(p) for p in parents])
        self._colors = (C.c_uint8 * (3 * J))(*color_table(J).reshape(-1).tolist())
        self._right = (C.c_int32 * max(len(right), 1))(*[int(j) for j in right])
        self._n_right = len(right)

    @property
    def frame_shape(self):
        return (self.S, self.S * (1 + self.panels), 3)

    def _range(self, frames):
        if frames is None:
            return 0, self.n_frames
        if isinstance(frames, (range, slice)):
            start, stop, step = frames.start or 0, frames.stop, 1 if frames.step is None else frames.step
            stop = self.n_frames if stop is None else stop
        else:
            start, stop = frames
            step = 1
        if step != 1 or not 0 <= start <= stop <= self.n_frames:
            raise GastError('render: frames %r is not a contiguous range within [0, %d)' % (frames, self.n_frames))
        return int(start), int(stop)

    def render(self, frames=None, out=None):
        """frames [f0, f1) (a range, a slice or a pair; None = all) as a CUDA uint8 tensor (F, S, S*(1+P), 3);
        `out`, when given, is a contiguous CUDA uint8 tensor of at least that size that receives them"""
        f0, f1 = self._range(frames)
        shape = (f1 - f0,) + self.frame_shape
        if out is None:
            out = torch.empty(shape, dtype=torch.uint8, device=self.device)
        else:
            if out.dtype != torch.uint8 or out.device != self.device or not out.is_contiguous() or \
                    out.numel() < int(np.prod(shape)):
                raise GastError('render: out must be a contiguous uint8 tensor on %s of %s' % (self.device, shape))
            out = out.view(-1)[:int(np.prod(shape))].view(shape)
        if f1 > f0:
            v = self.video
            with torch.cuda.device(self.device):
                _check(L.load().gast_render_frames(
                    _p(self.keypoints), int(self.keypoints.shape[0]), self.M, self.J, _p(self.poses),
                    int(self.poses.shape[0]), int(self.poses.shape[1]), _p(v), int(v.shape[0]) if v is not None else 0,
                    self.Hin, self.Win, self._parents, self._colors, self._right, self._n_right, self.n_bones, self.S,
                    self.dpi, ELEV, self.azim, RADIUS, DIST, self.flags, f0, f1 - f0, _p(out),
                    C.c_void_p(_stream(self.device))), 'gast_render_frames')
        return out


def render_frames(keypoints, poses, skeleton, azim, viewport, size=5, dpi=100, input_frames=None,
                  com_reconstrcution=False, limit=-1, downsample=1, input_video_skip=0, frames=None,
                  keypoints_metadata=None, follow_root=False):
    """The animation frames render_animation draws (vis_h36m.py:58-249), as a CUDA uint8 tensor (F, S, S*(1+P), 3)
    with S = size * dpi.

    keypoints (T, M, J, 2) or (T, J, 2) in image pixels; poses a dict (as the reference's) or list of (T, J, 3) world
    poses, one 3D panel each, or one shared panel for two persons with com_reconstrcution; skeleton: its parents()
    (and joints_right() when keypoints_metadata, the reference's dict, is not given: the right joints' discs are red);
    azim: the view's azimuth in degrees; viewport (w, h): the black image's size when there is no video;
    input_frames (T, H, W, 3) uint8: the decoded video from its first frame.  limit, downsample and input_video_skip
    as the reference applies them; frames: the range of the resulting frames to render (None = all).  follow_root
    centres each 3D panel on its pose's root (visualization.py:166-167).  Numpy arrays or CUDA tensors; no host
    synchronisation."""
    scene = Scene(keypoints, poses, skeleton, azim, viewport, size=size, dpi=dpi, input_frames=input_frames,
                  com_reconstrcution=com_reconstrcution, limit=limit, downsample=downsample,
                  input_video_skip=input_video_skip, keypoints_metadata=keypoints_metadata, follow_root=follow_root)
    return scene.render(frames)


# ------------------------------------------------------------------------------------------------
# render_animation's .mp4 output: the frames in chunks, piped to ffmpeg as raw RGB
# ------------------------------------------------------------------------------------------------
def _tool(name, why):
    exe = shutil.which(name)
    if exe is None:
        raise GastError('render_animation: %s was not found on PATH; it is needed %s' % (name, why))
    return exe


def _probe(path, entry):
    out = subprocess.run([_tool('ffprobe', 'to read ' + path), '-v', 'error', '-select_streams', 'v:0',
                          '-show_entries', 'stream=' + entry, '-of', 'csv=p=0', path], stdout=subprocess.PIPE,
                         check=True).stdout.decode().strip().splitlines()[0]
    return out


def read_video(path):
    """every frame of the video at path as (T, H, W, 3) uint8, decoded by ffmpeg as the reference's read_video does
    (vis_h36m.py:30-50, without its skip and limit: render_frames applies them)"""
    w, h = [int(v) for v in _probe(path, 'width,height').split(',')]
    cmd = [_tool('ffmpeg', 'to decode ' + path), '-v', 'error', '-i', path, '-f', 'image2pipe', '-pix_fmt', 'rgb24',
           '-vsync', '0', '-vcodec', 'rawvideo', '-']
    data = subprocess.run(cmd, stdout=subprocess.PIPE, check=True).stdout
    n = len(data) // (w * h * 3)
    return np.frombuffer(data, dtype=np.uint8, count=n * h * w * 3).reshape(n, h, w, 3)


def video_fps(path):
    a, b = _probe(path, 'r_frame_rate').split('/')
    return int(a) / int(b)


def write_mp4(scene, output, fps, bitrate, chunk=32):
    """every frame of scene encoded into output by ffmpeg (h264, yuv420p, bitrate in kbit/s, as matplotlib's ffmpeg
    writer asks for): chunks of frames rendered on the device, copied to pinned memory and piped as raw RGB while the
    next chunk renders.  Waits for ffmpeg to exit; a failure kills it."""
    exe = _tool('ffmpeg', 'to write ' + output)
    H, W, _ = scene.frame_shape
    cmd = [exe, '-y', '-v', 'error', '-f', 'rawvideo', '-pix_fmt', 'rgb24', '-s', '%dx%d' % (W, H), '-r', repr(float(fps)),
           '-i', '-', '-vcodec', 'h264', '-pix_fmt', 'yuv420p', '-b:v', '%dk' % int(bitrate), output]
    n = scene.n_frames
    chunk = max(1, min(int(chunk), n))
    shape = (chunk,) + scene.frame_shape
    bufs = [torch.empty(shape, dtype=torch.uint8, device=scene.device) for _ in range(2)]
    host = torch.empty(shape, dtype=torch.uint8, pin_memory=True)
    proc = subprocess.Popen(cmd, stdin=subprocess.PIPE)
    try:
        cur = scene.render((0, min(chunk, n)), out=bufs[0]) if n else None
        for k, f0 in enumerate(range(0, n, chunk)):
            m = int(cur.shape[0])
            host[:m].copy_(cur)                                  # waits for this chunk only
            nxt_f0 = f0 + chunk
            if nxt_f0 < n:                                       # the next chunk renders while this one is written
                cur = scene.render((nxt_f0, min(nxt_f0 + chunk, n)), out=bufs[(k + 1) % 2])
            proc.stdin.write(memoryview(host[:m].numpy()).cast('B'))
        proc.stdin.close()
        rc = proc.wait()
    except BaseException:
        proc.kill()
        proc.wait()
        raise
    if rc != 0:
        raise GastError('render_animation: ffmpeg exited with status %d writing %s' % (rc, output))


def render_animation(keypoints, keypoints_metadata, poses, skeleton, fps, bitrate, azim, output, viewport, limit,
                     downsample, size, input_video_path, input_video_skip, com_reconstrcution=False, follow_root=False,
                     bones_2d=None):
    """the body of both reference render_animation functions: .mp4 output only (a .gif is left to the caller, who can
    encode render_frames' frames), ffmpeg required; input_video_path is decoded by ffmpeg"""
    if output.endswith('.gif'):
        raise GastError('render_animation: .gif output is not supported; encode the frames of '
                        'gast_b200.render.render_frames instead')
    if not output.endswith('.mp4'):
        raise ValueError('Unsupported output format (only .mp4 and .gif are supported)')
    _tool('ffmpeg', 'to write ' + output)
    frames = None
    if input_video_path is not None:
        frames = read_video(input_video_path)
        if fps is None:
            fps = video_fps(input_video_path)
    scene = Scene(keypoints, poses, skeleton, azim, viewport, size=size, input_frames=frames,
                  com_reconstrcution=com_reconstrcution, limit=limit, downsample=downsample,
                  input_video_skip=input_video_skip, keypoints_metadata=keypoints_metadata, follow_root=follow_root,
                  bones_2d=bones_2d)
    if downsample > 1:
        fps /= downsample
    write_mp4(scene, output, fps, bitrate)
