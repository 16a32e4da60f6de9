"""Frame-by-frame causal lifting of many concurrent keypoint streams (SURVEY.md §8f N4).

The reference's real-time model is a causal `SpatioTemporalModelOptimized1f` fed the last `receptive_field`
frames of one stream for every new frame (`gen_skes.py:43-69`, `tools/inference.py:19-110`): O(rf) work per
frame.  `CausalStream` produces the same poses with O(1) work per frame: the library keeps, per temporal stage, a
ring of that stage's past inputs for all streams (`csrc/stream.cuh`, C ABI `gast_stream_push`), so a pushed frame
computes one new position per layer.  A stream's first frame stands for its whole (edge-padded) history exactly
like `UnchunkedGenerator(pad, causal_shift=pad)` does (`common/generators.py:210-221`).

The rings hold activations computed with the weights of the pushes that wrote them.  Any change to the model's
parameters or buffers (`load_state_dict`, an optimiser step, a training forward, which moves the BatchNorm running
statistics) therefore invalidates the history of every stream: the next push raises `GastError` unless `reset()`
(every stream) was called after the change.  Switching the GEMM core (`engine.set_gemm_core`) changes no weight and
keeps the streams.

`WindowStream` is the generic form for any callable network: a device ring of the last `rf` input frames and one
window forward per pushed frame (what the reference does; used for non-GAST callables and as the cross-check).
"""
import ctypes as C
import torch

from . import _lib as L


class CausalStream(object):
    """O(1)-per-frame lifting of `n_streams` concurrent streams with a causal model of the drop-in classes
    (`SpatioTemporalModelOptimized1f(causal=True)` as gen_skes.load_model_realtime builds it, or the dilated
    `SpatioTemporalModel(causal=True)`: the weights are interchangeable)."""

    def __init__(self, model_pos, n_streams, device=None):
        from . import engine
        if not getattr(model_pos, '_gast_causal', False):
            raise engine.GastError('CausalStream needs a causal model (gen_skes.py:59 builds it with causal=True)')
        if device is None:
            device = next(model_pos.parameters()).device
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise engine.GastError('CausalStream: the model must be on a CUDA device (there is no CPU path)')
        self.model = model_pos
        self.engine = engine
        self.rf = int(model_pos.receptive_field())
        self.n = int(n_streams)
        self.J = int(model_pos.num_joints_in)
        self.F = int(model_pos.in_features)
        self.step = 0
        self.fresh = torch.ones(self.n, dtype=torch.int32, device=self.device)     # every stream starts anew
        self._any_fresh = True
        self._all_fresh = True           # host-side: every stream starts anew at the next push (no device sync)
        self._sig = None                 # the handle's parameter signature at the last push
        self._state = None
        self._ws = None

    def reset(self, streams=None):
        """Forget the history of all (or the listed) streams: their next frame starts a new sequence."""
        if streams is None:
            self.fresh.fill_(1)
            self._all_fresh = True
        else:
            self.fresh[torch.as_tensor(streams, device=self.device, dtype=torch.long)] = 1
        self._any_fresh = True

    def push(self, frame):
        """frame (n_streams, J, in_features): the newest 2D keypoints of every stream (normalised screen
        coordinates).  Returns the 3D pose of that frame, (n_streams, J, 3)."""
        eng = self.engine
        frame = torch.as_tensor(frame, dtype=torch.float32, device=self.device).contiguous()
        assert frame.shape == (self.n, self.J, self.F), frame.shape
        if self.model.training:
            raise eng.GastError('CausalStream: call .eval() on the model (streaming is inference)')
        h = eng.model_handle(self.model, self.device)
        lib = h.lib
        y = torch.empty((self.n, self.J, 3), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            h.refresh(self.model, st)
            if self._sig is not None and h.sig != self._sig and not self._all_fresh:
                raise eng.GastError('CausalStream: the model\'s parameters or buffers changed since the last push '
                                    '(load_state_dict, an optimiser step or a training forward); the streams\' history '
                                    'was computed with the old weights -- call reset() before pushing again')
            if self._state is None:
                nb = lib.gast_stream_state_bytes(h.h, self.n)
                wb = lib.gast_stream_workspace_bytes(h.h, self.n)
                if nb == 0 or wb == 0:
                    raise eng.GastError('gast_stream_state_bytes: %s' % L.last_error())
                self._state = torch.empty(int(nb), dtype=torch.uint8, device=self.device)
                self._ws = torch.empty(int(wb), dtype=torch.uint8, device=self.device)
            fresh = self.fresh.data_ptr() if self._any_fresh else None
            rc = lib.gast_stream_push(h.h, C.c_void_p(self._state.data_ptr()), C.c_int64(self.step),
                                      C.c_void_p(frame.data_ptr()), C.c_void_p(y.data_ptr()), self.n,
                                      C.c_void_p(fresh), C.c_void_p(self._ws.data_ptr()), self._ws.numel(),
                                      C.c_void_p(st))
            if rc != 0:
                raise eng.GastError('gast_stream_push: %s' % L.last_error())
            if self._any_fresh:
                self.fresh.zero_()                       # (stream-ordered after the push that read it)
                self._any_fresh = False
                self._all_fresh = False
            self._sig = h.sig
        self.step += 1
        self.last_launches = int(lib.gast_last_launch_count(h.h))
        return y


class WindowStream(object):
    """Generic frame-by-frame driver for any window network `net((n, rf, J, F)) -> (n, T_out, J, 3)`: keeps the last
    `rf` frames of `n_streams` streams in one device tensor used as a ring and runs one window forward per pushed
    frame (O(rf) per frame, as the reference's real-time loop does)."""

    def __init__(self, net, n_streams, device=None):
        self.model = net
        self.rf = int(net.receptive_field())
        if device is None:
            device = next(net.parameters()).device
        self.device = torch.device(device)
        self.n = int(n_streams)
        self.J = int(net.num_joints_in)
        self.F = int(net.in_features)
        # ring[:, (head + k) % rf] is the k-th oldest frame of the window; `window` is its unrolled copy
        self.ring = torch.zeros((self.n, self.rf, self.J, self.F), dtype=torch.float32, device=self.device)
        self.window = torch.empty_like(self.ring)
        self.head = 0
        self.started = torch.zeros(self.n, dtype=torch.bool, device=self.device)

    def reset(self, streams=None):
        if streams is None:
            self.started.zero_()
        else:
            self.started[torch.as_tensor(streams, device=self.device)] = False

    def push(self, frame):
        frame = torch.as_tensor(frame, dtype=torch.float32, device=self.device)
        assert frame.shape == (self.n, self.J, self.F), frame.shape
        fresh = ~self.started
        if bool(fresh.any()):
            # a stream's first frame fills its whole window: the edge padding of generators.py:217-221
            self.ring[fresh] = frame[fresh].unsqueeze(1)
            self.started |= fresh
        self.ring[:, self.head] = frame                      # overwrite the oldest slot
        self.head = (self.head + 1) % self.rf
        k = self.rf - self.head                              # unroll: oldest frame first, newest last
        self.window[:, :k] = self.ring[:, self.head:]
        self.window[:, k:] = self.ring[:, :self.head]
        with torch.no_grad():
            return self.model(self.window)[:, -1]
