"""Live camera frames to placed 3D poses, one tick for C cameras at a time (DESIGN.md §8.10).

`LiveTick` is the reference's live path, `gen_img_kpts` (lib/pose/hrnet/pose_estimation/gen_kpts.py:115-175) feeding
the causal real-time models (gen_skes.py:43-69 load_model_realtime) and `revise_skes_real_time`
(tools/preprocess.py:158-172), for C cameras of one frame size with up to num_person tracked persons each:

    tick = LiveTick(det_net, pose_net, model_pos, cameras=C, frame_size=(W, H), num_person=2)
    out = tick(frames)          # frames (C, H, W, 3) uint8 on the device
    out.poses, out.keypoints, out.scores, out.ids, out.active

A tick is gast_letterbox -> det_net(batch, True) -> gast_person_detections -> gast_sort_update (one frame per camera,
empty frames skipped) -> gast_live_slots -> gast_person_crops of all C * num_person slots -> pose_net(crops) ->
gast_heatmap_decode -> gast_live_inputs -> [gast_tta_prepare] -> gast_stream_push_device -> [gast_tta_merge] ->
gast_camera_to_world(rot) -> gast_live_place, on static buffers and the caller's stream, with no host synchronisation.
Every slot is cropped and decoded every tick, empty or not: the fixed batch is what makes the tick one CUDA graph
(graph=True), at the cost of the nets' work for the empty slots.

A slot is bound to a SORT id, not to a row of SORT's output: a selected id that holds a slot keeps it, so two persons
who swap rows keep their histories.  The other selected ids take the free slots, then the slots not selected this
tick that were seen longest ago; a slot whose id changes restarts its stream.  A slot whose id is not selected this
tick is inactive, keeps its id, and its stream continues where it left off when the id comes back.

The stream pool is a `GraphedPoseStream` of C * num_person streams: its state set-up, library-stream layout, weight-
change rule and precision handling are that class's; its masks and input row are written on the device.
"""
import ctypes as C

import numpy as np
import torch

from . import detection as Dt
from . import keypoints2d as K
from .engine import GastError, _call, _p
from .realtime import GraphedPoseStream
from .tracking import SKIP_EMPTY, DeviceSort, status_message

ROT = (0.14070565, -0.15007018, -0.7552408, 0.62232804)     # tools/inference.py:16, the placement's camera rotation
MAX_PERSON = 32                                              # gast_live_slots: one lane per slot
STATUS_WORDS, STATUS_BITS = 16, 12                           # per camera: word, ticks, first tick of bits 0 .. 11
BOOK_INIT = (-1, -1, 1)                                      # a slot's id, last tick seen, restart flag
_REC_MESSAGES = ((K.REC_TRACKS, 'a frame with between 2 and num_person - 1 tracks (the reference cannot reshape them), '
                                'or a count outside -1 .. capacity'),
                 (K.REC_NONFINITE, 'a box that is not finite'),
                 (K.REC_EMPTY, 'a box with a non-positive width and height'),
                 (K.REC_MATRIX, 'forward matrices that are not finite'))


class LiveOutput(object):
    """A tick's outputs, static device tensors the next tick overwrites: poses (C, P, 17, 3) placed, zero in inactive
    slots; keypoints (C, P, 17, 2) H36M keypoints in pixels after the repair; scores (C, P, 17); ids (C, P) int64, the
    id SORT's rows give the person holding the slot (KalmanBoxTracker.id + 1, gen_img_kpts' human index), -1 if none
    ever did; active (C, P) bool."""

    def __init__(self, poses, keypoints, scores, ids, active):
        self.poses, self.keypoints, self.scores, self.ids, self.active = poses, keypoints, scores, ids, active


class LiveTick(GraphedPoseStream):
    """One tick for `cameras` cameras of frame_size (W, H): their frames in, the placed 3D pose of every tracked
    person out (module docstring).  det_net(batch, True) and pose_net(crops) are the caller's Darknet and HRNet, called
    as detection.video_boxes and keypoints2d.video_keypoints call them; both are called once at construction on zero
    inputs, which learns the heatmap size.  confidence and inp_dim are gen_kpts.py's --thred-score and --det-dim
    defaults, the symmetry lists tools/inference.py's.  With graph=True the first tick runs eagerly and everything
    after the copy into the static frame buffer `frames` is then captured as one CUDA graph, the caller's nets
    included; a net that cannot be captured is refused at construction.

    Refused with GastError before any launch: a non-causal model, a model in training mode and what PoseStream
    refuses, frames of another shape, dtype or device, and export_streams / import_streams / push / peek.  A tick
    never waits for the device; `status()` is the one call that does.  Weight and precision changes follow
    GraphedPoseStream's rule (graph=True) or PoseStream's (eager): after a change every camera must be reset()."""

    def __init__(self, det_net, pose_net, model_pos, cameras, frame_size, num_person=1, inp_dim=416, confidence=0.7,
                 nms_thresh=0.4, max_det=Dt.MAX_DET, max_age=1, min_hits=3, capacity=256, augment=False,
                 kps_left=None, kps_right=None, joints_left=None, joints_right=None, rgb_input=False, graph=False,
                 device=None):
        name = 'LiveTick'
        if hasattr(model_pos, '_gast_causal') and not model_pos._gast_causal:
            raise GastError('%s needs a causal model (gen_skes.py:43-69 load_model_realtime builds it with causal=True): '
                            'a non-causal model returns each pose latency ticks late' % name)
        if getattr(model_pos, 'training', False):
            raise GastError('%s: call .eval() on the model (streaming is inference)' % name)
        if hasattr(model_pos, 'num_joints_in') and (int(model_pos.num_joints_in) != 17 or int(model_pos.in_features) != 2):
            raise GastError('%s: the model must lift 17 joints of 2 features (got %d, %d)'
                            % (name, int(model_pos.num_joints_in), int(model_pos.in_features)))
        self.C, self.persons = int(cameras), int(num_person)
        if self.C < 1 or not 1 <= self.persons <= MAX_PERSON:
            raise GastError('%s: cameras >= 1 and 1 <= num_person <= %d expected (got %d, %d)'
                            % (name, MAX_PERSON, self.C, self.persons))
        self.W, self.H = int(frame_size[0]), int(frame_size[1])
        if not (0 < self.W <= K.MAX_SIDE and 0 < self.H <= K.MAX_SIDE):
            raise GastError('%s: a %d x %d frame (each side 1 .. %d)' % (name, self.W, self.H, K.MAX_SIDE))
        self.D = Dt.check_inp_dim(inp_dim)
        self._nw, self._nh = Dt.letterbox_geometry(self.W, self.H, self.D)
        if self._nw <= 0 or self._nh <= 0:
            raise GastError('%s: a %d x %d frame letterboxes to %d x %d' % (name, self.W, self.H, self._nw, self._nh))
        self.max_det = int(max_det)
        if self.max_det < 1:
            raise GastError('%s: max_det must be >= 1' % name)
        self.confidence, self.nms_thresh = float(np.float32(confidence)), float(np.float32(nms_thresh))
        self.rgb_input, self.use_graph = bool(rgb_input), bool(graph)
        super(LiveTick, self).__init__(model_pos, self.C * self.persons, augment=augment, kps_left=kps_left,
                                       kps_right=kps_right, joints_left=joints_left, joints_right=joints_right,
                                       device=device, K=1, peek=0)
        self.det_net, self.pose_net = det_net, pose_net
        C_, n, dev = self.C, self.n, self.device
        self.sort = DeviceSort(C_, max_age, min_hits, capacity, device=dev)
        self.capacity = self.sort.capacity
        f32, i32, i64 = (dict(dtype=t, device=dev) for t in (torch.float32, torch.int32, torch.int64))
        self.frames = torch.zeros((C_, self.H, self.W, 3), dtype=torch.uint8, device=dev)
        self._batch = torch.zeros((C_, 3, self.D, self.D), **f32)
        self._sizes = torch.tensor([[self.W, self.H]] * C_, **i32)
        self._boxes = torch.zeros((C_, self.max_det, 4), **f32)
        self._box_scores = torch.zeros((C_, self.max_det), **f32)
        self._counts = torch.zeros(C_, **i32)
        self._rows = torch.zeros((C_, 1, self.capacity, 5), dtype=torch.float64, device=dev)
        self._track_counts = torch.zeros((C_, 1), **i32)
        self._sort_status = torch.zeros(C_, **i32)
        self._book = torch.tensor(BOOK_INIT, **i64)[:, None].repeat(1, n).contiguous()    # (3, C * P)
        self._status = torch.full((C_, STATUS_WORDS), -1, **i64)
        self._status[:, :2] = 0
        self._slot_active = torch.zeros(n, **i32)
        self._fwd = torch.zeros((n, 6), dtype=torch.float64, device=dev)
        self._inv = torch.zeros((n, 6), dtype=torch.float64, device=dev)
        self._cs = torch.zeros((n, 4), **f32)
        self._frame_index = torch.arange(n, **i32) // self.persons
        w, h = K.IMAGE_SIZE
        self._crops = torch.zeros((n, 3, h, w), **f32)
        self._preds = torch.zeros((n, 17, 2), **f32)
        self._maxvals = torch.zeros((n, 17, 1), **f32)
        self._kpts = torch.zeros((n, 17, 2), **f32)
        self._scores = torch.zeros((n, 17), **f32)
        self._active = torch.zeros(n, dtype=torch.uint8, device=dev)
        self._world = torch.zeros((n, 17, 3), **f32)
        self._poses = torch.zeros((n, 17, 3), **f32)
        self._q = (C.c_float * 4)(*ROT)
        self._t = (C.c_float * 3)(0.0, 0.0, 0.0)
        self.out = LiveOutput(self._poses.view(C_, self.persons, 17, 3), self._kpts.view(C_, self.persons, 17, 2),
                              self._scores.view(C_, self.persons, 17), self._book[0].view(C_, self.persons),
                              self._active.view(torch.bool).view(C_, self.persons))
        self._probe_nets()

    # ---- construction -------------------------------------------------------------------------------------------
    def _det(self):
        pred = self.det_net(self._batch, True)
        N = Dt.num_predictions(self.D)
        if not isinstance(pred, torch.Tensor) or not pred.is_cuda or pred.dtype != torch.float32 or \
                tuple(pred.shape) != (self.C, N, Dt.ATTRS):
            raise GastError('LiveTick: the detector must return (%d, %d, %d) float32 predictions on the device'
                            % (self.C, N, Dt.ATTRS))
        return pred.contiguous()

    def _pose(self):
        heat = self.pose_net(self._crops)
        if not isinstance(heat, torch.Tensor) or not heat.is_cuda or heat.dtype != torch.float32 or heat.dim() != 4 \
                or int(heat.shape[0]) != self.n or int(heat.shape[1]) != 17:
            raise GastError('LiveTick: the pose net must return (%d, 17, hh, hw) float32 heatmaps on the device' % self.n)
        hm = (int(heat.shape[3]), int(heat.shape[2]))
        if getattr(self, '_hm', hm) != hm:
            raise GastError('LiveTick: the pose net returned %d x %d heatmaps, %d x %d at construction'
                            % (hm + self._hm))
        return heat.contiguous()

    def _probe_nets(self):
        """call both nets once on the zero buffers: the heatmap size, and with graph=True a trial capture"""
        with torch.cuda.device(self.device), torch.no_grad():
            self._det()
            heat = self._pose()
            self._hm = (int(heat.shape[3]), int(heat.shape[2]))
            if not (0 < self._hm[0] <= K.MAX_HEATMAP and 0 < self._hm[1] <= K.MAX_HEATMAP):
                raise GastError('LiveTick: %d x %d heatmaps (sides <= %d)' % (self._hm + (K.MAX_HEATMAP,)))
            if self.use_graph:
                try:
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._det()
                        self._pose()
                    del g
                except GastError:
                    raise
                except Exception as e:
                    raise GastError('LiveTick: the detector or the pose net cannot be captured in a CUDA graph: %s'
                                    % e) from e

    # ---- the tick -----------------------------------------------------------------------------------------------
    def _run(self, h, st):
        """enqueue one tick after the frame copy on stream `st` -> the library's launch count (the nets excluded)"""
        C_, n, P = self.C, self.n, self.persons
        s = C.c_void_p(st)
        w, hh_ = K.IMAGE_SIZE
        hw, hh = self._hm
        _call('gast_letterbox', _p(self.frames), C_, self.H, self.W, self.D, self._nw, self._nh,
              Dt.RGB_INPUT if self.rgb_input else 0, _p(self._batch), s)
        with torch.no_grad():
            pred = self._det()
        _call('gast_person_detections', _p(pred), C_, int(pred.shape[1]), Dt.ATTRS, self.D, _p(self._sizes),
              self.confidence, self.nms_thresh, self.max_det, 0, _p(self._boxes), _p(self._box_scores),
              _p(self._counts), None, None, s)
        _call('gast_sort_update', _p(self.sort.state), C_, self.capacity, 1, _p(self._boxes), _p(self._counts),
              self.max_det, SKIP_EMPTY, _p(self._rows), _p(self._track_counts), _p(self._sort_status), s)
        _call('gast_live_slots', _p(self._rows), _p(self._track_counts), _p(self._sort_status), C_, self.capacity, P,
              self.W, self.H, w, hh_, hw, hh, _p(self._book), _p(self._status), _p(self._slot_active), _p(self._fwd),
              _p(self._inv), _p(self._cs), s)
        flags = (K.RGB_INPUT if self.rgb_input else 0) | K.NET_ORDER
        _call('gast_person_crops', _p(self.frames), C_, self.H, self.W, _p(self._frame_index), _p(self._fwd), n, w, hh_,
              flags, _p(self._crops), s)
        with torch.no_grad():
            heat = self._pose()
        _call('gast_heatmap_decode', _p(heat), _p(self._inv), n, 17, hh, hw, 1, _p(self._preds), _p(self._maxvals), s)
        N = self.copies * n
        _call('gast_live_inputs', _p(self._preds), _p(self._maxvals), _p(self._slot_active), n, self.W, self.H,
              self.copies, _p(self._book[2]), _p(self._kpts), _p(self._scores), _p(self._x), _p(self._mask_dev[:N]),
              _p(self._mask_dev[N:2 * N]), _p(self._active), s)
        launches = 9 + self._tick(h, st)
        _call('gast_camera_to_world', _p(self._y), _p(self._world), n * 17, self._q, self._t, s)
        _call('gast_live_place', _p(self._world), _p(self._kpts), _p(self._active), C_, P, float(self.W),
              _p(self._poses), s)
        return launches

    def _eager(self, h, st):
        """refresh the handle, refuse stale history, allocate the state and the workspace, run one tick eagerly"""
        self._begin(h, st)
        wb = self.engine._check_size(h.lib.gast_stream_device_workspace_bytes(h.h, self.copies * self.n, 1),
                                     'gast_stream_device_workspace_bytes')
        if self._ws is None or self._ws.numel() < wb:
            self._ws = torch.empty(wb, dtype=torch.uint8, device=self.device)
        return self._run(h, st)

    def __call__(self, frames):
        """frames (C, H, W, 3) uint8 on the tick's device -> `out` (LiveOutput), overwritten by the next tick"""
        eng, name = self.engine, 'LiveTick'
        if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.device == self.device and
                frames.dtype == torch.uint8 and tuple(frames.shape) == tuple(self.frames.shape)):
            raise GastError('%s: frames (%d, %d, %d, 3) uint8 on %s expected, got %s' % (
                name, self.C, self.H, self.W, self.device,
                (tuple(frames.shape), getattr(frames, 'dtype', None), getattr(frames, 'device', None))))
        if self.model.training:
            raise GastError('%s: call .eval() on the model (streaming is inference)' % name)
        with torch.cuda.device(self.device):
            now = eng.param_sig(self.model)
            if self.graph is not None:
                if self._mode_now() != self._mode:
                    raise GastError('%s: engine.set_precision or engine.set_gemm_core changed since the tick was '
                                    'captured; construct a new %s' % (name, name))
                if now != self._sig or self._h.sig != self._sig:
                    self._refuse_stale(self._sig, now)
                    self.graph = None
            else:
                self._refuse_stale(self._sig, now)
            st = torch.cuda.current_stream(self.device).cuda_stream
            if frames.data_ptr() != self.frames.data_ptr():
                self.frames.copy_(frames, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
                launches = self._launches
            else:
                h = eng.model_handle(self.model, self.device)
                launches = self._eager(h, st)
                self._h, self._sig = h, h.sig
                if self.use_graph:
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        self._launches = self._run(h, torch.cuda.current_stream(self.device).cuda_stream)
                    self.graph, self._mode = graph, self._mode_now()
        self.book.fresh[:] = False
        self.last_launches = launches
        return self.out

    # ---- status and reset ---------------------------------------------------------------------------------------
    def status(self):
        """-> (words (C,), first (C, 12)) int64 numpy: each camera's sticky status word (SORT's bits or'ed with
        keypoints2d.REC_*) and the tick that first set each of its bits 0 .. 11 (-1 for none).  One copy to the host:
        the only call of this class that waits for the device."""
        st = self._status.cpu().numpy()
        return st[:, 0].copy(), st[:, 2:2 + STATUS_BITS].copy()

    def check(self):
        """GastError for the first camera whose status word is set, with the host path's message"""
        words, first = self.status()
        bad = np.flatnonzero(words)
        if not bad.size:
            return
        c = int(bad[0])
        word = int(words[c])
        if word & K.SORT_BITS:
            raise GastError('tracking: sequence %d: %s' % (c, status_message(word & K.SORT_BITS)))
        for bit, what in _REC_MESSAGES:
            if word & bit:
                raise GastError('keypoints2d: camera %d tick %d: %s' % (c, int(first[c, bit.bit_length() - 1]), what))

    def reset(self, cameras=None):
        """Start the listed cameras (all for None) afresh: SORT re-initialised with the ids continuing from its next
        id, the slot book cleared, the status word cleared and every stream of those cameras restarting."""
        cams = np.arange(self.C) if cameras is None else np.asarray(cameras, dtype=np.int64).reshape(-1)
        if cams.size and (cams.min() < 0 or cams.max() >= self.C or np.unique(cams).size != cams.size):
            raise GastError('LiveTick.reset: cameras must be distinct indices in [0, %d) (got %s)'
                            % (self.C, cams.tolist()))
        srt = self.sort
        with torch.cuda.device(self.device):
            st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            next_ids = srt.header()[:, 1].clone()
            for c in cams.tolist():
                _call('gast_sort_init', C.c_void_p(srt.state.data_ptr() + c * srt.state_bytes), 1, self.capacity,
                      srt.max_age, srt.min_hits, C.c_void_p(next_ids[c:].data_ptr()), st)
                rows = slice(c * self.persons, (c + 1) * self.persons)
                for plane, v in enumerate(BOOK_INIT):
                    self._book[plane, rows].fill_(v)
                self._status[c, 0].fill_(0)
                self._status[c, 2:].fill_(-1)
        if cams.size:
            self.book.reset((cams[:, None] * self.persons + np.arange(self.persons)[None, :]).reshape(-1))

    # ---- refused ------------------------------------------------------------------------------------------------
    def push(self, frames, streams=None):
        raise GastError('LiveTick: call the tick with the camera frames; its streams are pushed on the device')

    def end(self, streams=None):
        raise GastError('LiveTick: live streams do not end; reset() the cameras to restart them')

    def export_streams(self, streams):
        raise GastError('LiveTick: moving live streams between pools is not supported')

    def import_streams(self, snapshot, streams):
        raise GastError('LiveTick: moving live streams between pools is not supported')
