"""Host glue between the drop-in nn.Module shells (model/*.py) and libgast_b200.so.

For each module instance (and device) the engine keeps one C handle.  The handle borrows
the module's own parameter/buffer storage (`gast_bind`, no copies), so optimiser steps and
`load_state_dict` are seen; derived constants are refreshed (`gast_prepare`) whenever a
tensor's (data_ptr, _version) signature changes.  torch provides device memory (outputs and
each call's workspace from the caching allocator) and the current CUDA stream -- plumbing only.  Every call orders all of
its work on the current stream and keeps no device buffer after it returns, so calls on several streams and inside a
user's CUDA graph capture behave as torch's own ops do.

No fallback: CPU tensors, a missing library or an unsupported mode raise.
"""
import ctypes as C
import math

import torch

from . import _lib as L

_FORCE_CORE = {'core': 0}   # 0 auto, 1 FFMA (A/B checks of the tensor-core core on the GPU)


def set_gemm_core(core):
    """0 = auto (tensor cores where the shape allows), 1 = FP32 FFMA core everywhere."""
    _FORCE_CORE['core'] = int(core)


class GastError(RuntimeError):
    pass


_PRECISIONS = {'fp32': 0, 'tf32': 1, 'fp16': 16}     # set_precision -> gast_set_precision's mode
_TRAIN_PRECISIONS = {'fp32': 0, 'tf32': 1}          # set_training_precision -> gast_set_train_precision's mode


def set_precision(module, mode):
    """Arithmetic of the tensor-core GEMMs of `module` and all of its sub-modules, like torch's `allow_tf32`:
    'fp32' (default) is fp32-grade (3xTF32, the reference's numbers to ~1e-7 relative); 'tf32' is one TF32 product
    per multiply-add with fp32 accumulation, faster and about 1e-3 relative off (DESIGN.md §4.1); 'fp16' is the
    arithmetic of a half model behind float32 input, parameters and poses: every activation stored in fp16, one fp16
    product per multiply-add with fp32 accumulation, fastest and about 2e-3 of max |y| off (DESIGN.md §4.1, "The fp16
    precision").  'tf32' and 'fp16' are for inference: forward under no_grad, run_model_chunked, run_model_mpjpe, the
    streams, lift_sequences, tta.evaluate_sequence; a train-mode forward or one that builds an autograd graph raises
    unless the training precision is 'tf32' (set_training_precision).  'fp16' runs whole float32 models with channels
    that are multiples of 32 on the tensor-core core; a half model (model.half()) raises at 'fp16' (it has its own
    fp16 arithmetic), as does a sub-module called on its own.  The streams keep their history in fp16 at 'fp16', so
    a PoseStream pool with history refuses a switch between 'fp16' and the other two (DESIGN.md §4.1).  The setting
    lives in each module's __dict__ (DataParallel replicas and deepcopies keep it, state_dict does not).  Returns the
    module."""
    if mode not in _PRECISIONS:
        raise GastError("set_precision: mode must be 'fp32', 'tf32' or 'fp16' (got %r)" % (mode,))
    for m in module.modules():
        m.__dict__['_gast_precision'] = mode
    return module


def get_precision(module):
    """'fp32', 'tf32' or 'fp16' (set_precision)"""
    return module.__dict__.get('_gast_precision', 'fp32')


def set_training_precision(module, mode):
    """Arithmetic of training and of every gradient of `module` and its sub-modules: 'fp32' (default) is fp32-grade;
    'tf32' runs every tensor-core GEMM of a train-mode forward, of the backward and of the eval-mode backward's
    recompute as one TF32 product, and the weight gradients whose N and K are multiples of 32 on a TF32 tensor-core
    kernel (DESIGN.md §4.3).  BatchNorm statistics, dropout and the remaining parameter gradients stay fp32; the
    results repeat bit for bit run to run and across CUDA-graph replays in either mode.  With 'tf32' the model trains
    and differentiates whatever set_precision says.  An eval-mode forward that builds an autograd graph is still the
    inference forward, at the inference precision (set_precision); its backward recomputes the activations at this
    precision.  Stored in each module's __dict__ like set_precision (DataParallel replicas and deepcopies keep it,
    state_dict does not).  Returns the module."""
    if mode not in _TRAIN_PRECISIONS:
        raise GastError("set_training_precision: mode must be 'fp32' or 'tf32' (got %r)" % (mode,))
    for m in module.modules():
        m.__dict__['_gast_train_precision'] = mode
    return module


def get_training_precision(module):
    """'fp32' or 'tf32' (set_training_precision)"""
    return module.__dict__.get('_gast_train_precision', 'fp32')


def _fp32_only(module, what):
    prec = get_precision(module)
    if prec != 'fp32' and get_training_precision(module) == 'fp32':
        raise GastError("%s: the model is set to %s, which is inference-only; call "
                        "engine.set_precision(model, 'fp32') to train or differentiate it"
                        % (what, 'TF32' if prec == 'tf32' else 'the fp16 precision'))


_HALF_ONLY = ('the model is half precision (model.half()), which runs inference only: the eval-mode forward under '
              'torch.no_grad() / torch.inference_mode() (model(x), run_model_chunked); call model.float() for %s')


def model_dtype(module, what):
    """torch.float32 or torch.float16, the floating dtype of all of the module's parameters and buffers: a model
    runs in half once model.half() made every one of them fp16.  A mix of dtypes, or any other, raises, as a torch
    module of mixed dtypes does."""
    dts = {v.dtype for _, v in named_tensors(module) if v.is_floating_point()}
    if not dts or dts == {torch.float32}:
        return torch.float32
    if dts == {torch.float16}:
        return torch.float16
    raise GastError("%s: the module's parameters and buffers must all be float32 or all float16 (model.float() / "
                    "model.half()), got %s" % (what, ', '.join(sorted(str(d) for d in dts))))


def refuse_half(module, what, instead):
    """raise when `module` is a half model: `what` runs in float32 only"""
    if any(v.dtype == torch.float16 for _, v in named_tensors(module)):
        raise GastError('%s: %s' % (what, _HALF_ONLY % instead))


def _check(rc, what):
    if rc != 0:
        raise GastError('%s: %s' % (what, L.last_error()))


def _check_size(n, what):
    """-> n, the result of a size entry (`*_bytes`, `*_floats`), as an int; 0 is that entry's refusal"""
    if n == 0:
        raise GastError('%s: %s' % (what, L.last_error()))
    return int(n)


def _mask_lists(m):
    idx = m.nonzero()        # row-major order == order of `e` (local_attention.py:25,41)
    rows = (C.c_int32 * len(idx))(*[int(i) for i in idx[:, 0]])
    cols = (C.c_int32 * len(idx))(*[int(i) for i in idx[:, 1]])
    return rows, cols, len(idx)


def _m2d(m):
    m = m.detach().cpu()
    return m[0] if m.dim() == 3 else m


def named_tensors(module):
    """(key, tensor) pairs under the names `module.state_dict()` uses, in its order: named_params with the persistent
    buffers.  Unlike state_dict() this also works on the per-forward replicas of nn.DataParallel (trainval.py:56-61),
    whose weights are broadcast views kept as plain attributes (`_former_parameters`) instead of in `_parameters`."""
    return named_params(module, buffers=True)


def named_params(module, buffers=False):
    """named_parameters() that also sees the broadcast parameter views of a DataParallel replica
    (they are non-leaf tensors connected to the real parameters, so autograd routes the gradients); with `buffers`
    each module's persistent buffers follow its parameters."""
    out = []
    for prefix, mod in module.named_modules():
        pre = prefix + '.' if prefix else ''
        former = getattr(mod, '_former_parameters', None) or {}
        for k, v in mod._parameters.items():
            if v is not None:
                out.append((pre + k, v))
        for k, v in former.items():
            if v is not None and mod._parameters.get(k) is None:
                out.append((pre + k, v))
        if buffers:
            for k, v in mod._buffers.items():
                if v is not None and k not in mod._non_persistent_buffers_set:
                    out.append((pre + k, v))
    return out


def param_sig(module):
    """the (data_ptr, _version) signature of the module's parameters and buffers (named_tensors): it changes whenever
    one of them is replaced or written in place"""
    return tuple((v.data_ptr(), v._version) for _, v in named_tensors(module))


class _HandleStore(dict):
    """device -> _Handle, kept in the module's __dict__ (so that the shallow-copied replicas of
    nn.DataParallel share it).  Native handles are per process and per device: a deepcopy / pickle of the
    module (EMA copies, torch.save(model)) gets an empty store and builds its own handles on first use."""

    def __deepcopy__(self, memo):
        return _HandleStore()

    def __reduce__(self):
        return (_HandleStore, ())


class _Handle(object):
    def __init__(self, module, kind, device, cfg_kw, sym=None, con=None):
        lib = L.load()
        self.lib = lib
        self.kind = kind
        self.device = device
        cfg = L.GastCfg()
        cfg.kind = kind
        cfg.device = device.index if device.index is not None else torch.cuda.current_device()
        for k, v in cfg_kw.items():
            if k == 'filter_widths':
                for i, fw in enumerate(v):
                    cfg.filter_widths[i] = int(fw)
                cfg.num_stages = len(v)
            else:
                setattr(cfg, k, int(v))
        keep = []
        if sym is not None:
            r, c, n = _mask_lists(_m2d(sym))
            cfg.sym_rows, cfg.sym_cols, cfg.sym_nnz = r, c, n
            keep += [r, c]
        if con is not None:
            r, c, n = _mask_lists(_m2d(con))
            cfg.con_rows, cfg.con_cols, cfg.con_nnz = r, c, n
            keep += [r, c]
        self.h = C.c_void_p()
        _check(lib.gast_create(C.byref(self.h), C.byref(cfg)), 'gast_create')
        self.sig = None
        self.core = None
        self.precision = 0
        self.train_precision = 0
        self.act_dtype = 0               # gast_set_activation_dtype: 1 (GAST_F16) for a half model
        self.f32 = None                  # a half model's float32 copies of its tensors, bound in their place

    def __del__(self):
        try:
            if getattr(self, 'h', None) and self.h.value:
                self.lib.gast_destroy(self.h)
                self.h = C.c_void_p()
        except Exception:
            pass

    def apply_core(self, module):
        """hand the set_gemm_core() choice and the module's set_precision() and set_training_precision() to the
        library handle (every forward, training or eval, and every stream push), and for a whole model its activation
        type: fp16 for a half model.  Half and the fp16 precision go off first and on last, as the library refuses
        TF32, the fp16 precision and the FFMA core in half, and half and the FFMA core at the fp16 precision.  A half
        model at 'fp16' raises here, before anything is set or launched."""
        act = 1 if self.kind == L.KIND_MODEL and model_dtype(module, 'forward') == torch.float16 else 0
        prec = _PRECISIONS[get_precision(module)]
        if act and prec == _PRECISIONS['fp16']:
            raise GastError("the model is half precision (model.half()), which has its own fp16 arithmetic; the fp16 "
                            "precision is for float32 models: call engine.set_precision(model, 'fp32') (or "
                            "model.float())")
        if act == 0 and self.act_dtype != 0:
            self._set_act(0)
        if self.precision == _PRECISIONS['fp16'] and prec != self.precision:
            self._set_precision(prec)
        if _FORCE_CORE['core'] != self.core:
            _check(self.lib.gast_set_gemm_core(self.h, _FORCE_CORE['core']), 'gast_set_gemm_core')
            self.core = _FORCE_CORE['core']
        if prec != self.precision:
            self._set_precision(prec)
        tprec = _TRAIN_PRECISIONS[get_training_precision(module)]
        if tprec != self.train_precision:
            _check(self.lib.gast_set_train_precision(self.h, tprec), 'gast_set_train_precision')
            self.train_precision = tprec
        if act != self.act_dtype:
            self._set_act(act)

    def _set_precision(self, prec):
        _check(self.lib.gast_set_precision(self.h, prec), 'gast_set_precision')
        self.precision = prec

    def _set_act(self, act):
        _check(self.lib.gast_set_activation_dtype(self.h, act), 'gast_set_activation_dtype')
        self.act_dtype = act

    def refresh(self, module, stream):
        """(re)bind + prepare when any parameter/buffer moved or changed."""
        sig = param_sig(module)
        self.apply_core(module)
        if sig == self.sig:
            return
        items = named_tensors(module)
        # a half model: the library folds float32 parameters, so float32 copies are bound (kept until the next change)
        self.f32 = [(k, v.float() if v.dtype == torch.float16 else v) for k, v in items] if self.act_dtype else None
        _bind(self, 'gast_bind', self.f32 or items)
        _check(self.lib.gast_prepare(self.h, C.c_void_p(stream)), 'gast_prepare')
        self.sig = sig

    def bind_only(self, module):
        """bind parameter/buffer storage without the eval-mode prepare (training path)"""
        self.apply_core(module)
        _bind(self, 'gast_bind', named_tensors(module))
        self.sig = None

    def forward(self, x, y, B, T, strided_now, stream, target=None, loss=None):
        """gast_forward, or with a target gast_forward_mpjpe, on a workspace of the call's own from the caching
        allocator, as the chunked forward, the backward and training take theirs.  It is freed to the current stream
        `stream` when the call returns, and the allocator hands it only to later work of that stream (or keeps it in
        the private pool of a graph being captured), so no call in flight on another stream or in a graph shares it."""
        need = _check_size(self.lib.gast_workspace_bytes(self.h, B, T, strided_now), 'gast_workspace_bytes')
        ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        tail = (B, T, strided_now, _p(ws), ws.numel(), C.c_void_p(stream))
        if target is None:
            _check(self.lib.gast_forward(self.h, _p(x), _p(y), *tail), 'gast_forward')
        else:
            _check(self.lib.gast_forward_mpjpe(self.h, _p(x), _p(target), _p(y), _p(loss), *tail),
                   'gast_forward_mpjpe')

    def launches(self):
        return int(self.lib.gast_last_launch_count(self.h))

    def wgrad_tc_launches(self):
        """weight gradients of the last training step or eval backward that ran on the TF32 tensor-core kernel"""
        return int(self.lib.gast_last_wgrad_tc_launch_count(self.h))


def _bind(handle, entry, items):
    """hand (key, tensor) pairs to the library entry `entry` (gast_bind or gast_bind_grads) of `handle`"""
    n = len(items)
    keys = (C.c_char_p * n)()
    ptrs = (C.c_void_p * n)()
    numel = (C.c_int64 * n)()
    for i, (k, v) in enumerate(items):
        if not v.is_cuda or v.device != handle.device:
            raise GastError('parameter %r is on %s, expected %s (call .cuda() on the module)'
                            % (k, v.device, handle.device))
        if not v.is_contiguous():
            raise GastError('parameter %r is not contiguous' % k)
        if v.is_floating_point() and v.dtype != torch.float32:
            raise GastError('parameter %r is %s: the library binds float32 tensors (a whole model in half precision binds '
                            'float32 copies; call .float() on a sub-module)' % (k, v.dtype))
        keys[i] = k.encode()
        ptrs[i] = v.data_ptr()
        numel[i] = v.numel()
    _check(getattr(handle.lib, entry)(handle.h, n, keys, ptrs, numel), entry)


def _p(t):
    """a tensor's device pointer for the C ABI (None: null)"""
    return C.c_void_p(t.data_ptr() if t is not None else None)


def _cuda_f32(x, what):
    """x as a contiguous CUDA float32 tensor; anything else raises (there is no CPU path)"""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise GastError('%s: input must be a CUDA tensor -- this implementation has no CPU path' % what)
    if x.dtype != torch.float32:
        raise GastError('%s: input must be float32 (got %s)' % (what, x.dtype))
    return x.contiguous()


def _cuda_input(x, dtype, what):
    """x as a contiguous CUDA tensor of the model's dtype (float32, or float16 for a half model); anything else raises"""
    if dtype == torch.float32:
        return _cuda_f32(x, what)
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise GastError('%s: input must be a CUDA tensor -- this implementation has no CPU path' % what)
    if x.dtype != dtype:
        raise GastError('%s: the model is %s, the input %s (convert one of them)' % (what, dtype, x.dtype))
    return x.contiguous()


def _ilist(v):
    """a host int32 array of the indices `v` (None: none) for the C ABI, and their count"""
    v = [] if v is None else list(v)
    return (C.c_int32 * max(len(v), 1))(*[int(i) for i in v]), len(v)


def _handle_for(module, device, factory):
    store = module.__dict__.get('_gast_handles')
    if store is None:
        store = module.__dict__.setdefault('_gast_handles', _HandleStore())
    key = (device.type, device.index)
    h = store.get(key)
    if h is None:
        h = factory()
        store[key] = h
    return h


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


class _TrainFn(torch.autograd.Function):
    """Training-mode forward/backward of the whole model on the CUDA library (gast_forward_train /
    gast_backward).  Parameters are passed as inputs so that autograd routes their gradients."""

    @staticmethod
    def forward(ctx, module, handle, x, names, *params):
        dev = x.device
        B, T = int(x.shape[0]), int(x.shape[1])
        lib = handle.lib
        with torch.cuda.device(dev):
            st = _stream(dev)
            handle.bind_only(module)
            need = _check_size(lib.gast_train_workspace_bytes(handle.h, B, T, C.c_float(float(module._gast_dropout))),
                               'gast_train_workspace_bytes')
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            y = _new_output(module, handle, B, T, 1 if module._gast_strided else 0, dev)
            p = float(module._gast_dropout)
            seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if p > 0 else 0
            # device-side dropout counter (set by a graph-capturing trainer): keeps the masks fresh across replays
            ds = module.__dict__.get('_gast_dropout_state')
            _check(lib.gast_set_dropout_state(handle.h, _p(ds)), 'gast_set_dropout_state')
            _check(lib.gast_forward_train(handle.h, _p(x), _p(y), B, T, C.c_float(p), C.c_uint64(seed), _p(ws),
                                          ws.numel(), C.c_void_p(st)), 'gast_forward_train')
        # BatchNorm bookkeeping that torch does in Python: num_batches_tracked (this also bumps the
        # buffers' versions, so the eval-mode constants are refreshed on the next eval forward)
        with torch.no_grad():
            nbt = [mod.num_batches_tracked for mod in module.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
            if nbt:
                torch._foreach_add_(nbt, 1)              # one launch instead of one per BatchNorm
        handle.sig = None
        ctx.handle, ctx.ws, ctx.names, ctx.params = handle, ws, names, params
        ctx.direct = bool(module.__dict__.get('_gast_direct_grads', False))
        ctx.x = x            # the backward re-reads the input (init_bn statistics): keep it alive
        ctx.dev = dev
        return y

    @staticmethod
    def backward(ctx, dy):
        handle, ws, names, params = ctx.handle, ctx.ws, ctx.names, ctx.params
        lib = handle.lib
        n = len(params)
        need_x = ctx.needs_input_grad[2]
        need_p = any(ctx.needs_input_grad[4:])
        # A trainer that owns the gradient buffers (module._gast_direct_grads, set by gast_b200.trainer: every .grad is
        # a view of its flat all-reduce buffer and one backward runs per step) gets the gradients WRITTEN straight into
        # them: autograd's AccumulateGrad would otherwise launch one add per parameter (166 per step at 27f/128ch,
        # 0.46 ms of a 8.3 ms step).  Everyone else gets them through autograd as usual.
        direct = ctx.direct and all(p.is_leaf and p.grad is not None and p.grad.is_contiguous() and
                                    p.grad.dtype == torch.float32 and p.grad.device == p.device and
                                    p.grad.shape == p.shape for p in params)
        dy = dy.contiguous()
        dx = torch.empty_like(ctx.x) if need_x else None
        with torch.cuda.device(ctx.dev):
            views = _bind_grad_views(handle, names, params, direct, ctx.dev) if need_p else None
            # no parameter needs a gradient (all frozen, only x is differentiated): the library skips every
            # weight-gradient kernel
            _check(lib.gast_backward_input(handle.h, _p(dy), _p(dx), 1 if need_p else 0, _p(ws), ws.numel(),
                                           C.c_void_p(_stream(ctx.dev))), 'gast_backward')
        ctx.ws = None
        ctx.x = None
        if direct or views is None:
            return (None, None, dx, None) + (None,) * n
        return (None, None, dx, None) + tuple(views)


def _bind_grad_views(handle, names, params, direct, dev):
    """bind one gradient buffer per parameter (gast_bind_grads): the parameters' own .grad when `direct`, else views of
    one fresh flat buffer, which are returned for autograd to accumulate"""
    flat = None if direct else torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
    views, off = [], 0
    for p in params:
        views.append(p.grad if direct else flat[off:off + p.numel()].view_as(p))
        off += p.numel()
    _bind(handle, 'gast_bind_grads', list(zip(names, views)))
    return views


class _EvalFn(torch.autograd.Function):
    """Eval-mode forward of the whole model with a backward (model.eval(): BatchNorm on the running statistics, no
    dropout), whole (max_frames None) or in passes of at most max_frames output positions.  The forward is the
    inference forward, unchanged.  The backward (gast_eval_backward, or gast_eval_backward_chunked pass by pass)
    recomputes the activations from the saved x with a frozen-BatchNorm training forward, then runs the training
    backward: nothing is held on the device between the two beyond x.  x, the parameters and the running statistics
    are saved with save_for_backward, so an in-place change to any of them before the backward raises torch's version
    error, as it does for the reference module."""

    @staticmethod
    def forward(ctx, module, handle, x, strided_now, max_frames, names, *params):
        y = _chunked_forward(module, handle, x, strided_now, max_frames)
        stats = [v for k, v in named_tensors(module) if k.endswith('.running_mean') or k.endswith('.running_var')]
        ctx.save_for_backward(x, *params, *stats)
        ctx.module, ctx.handle, ctx.sn, ctx.max_frames, ctx.names, ctx.n = (module, handle, strided_now, max_frames,
                                                                            names, len(params))
        return y

    @staticmethod
    def backward(ctx, dy):
        saved = ctx.saved_tensors
        x, params = saved[0], saved[1:1 + ctx.n]
        module, h, mf = ctx.module, ctx.handle, ctx.max_frames
        need_x = ctx.needs_input_grad[2]
        need_p = any(ctx.needs_input_grad[6:])
        dev = x.device
        B, T = int(x.shape[0]), int(x.shape[1])
        dy = dy.contiguous()
        with torch.cuda.device(dev):
            st = _stream(dev)
            h.refresh(module, st)            # binds the current storage and GEMM-core choice (no work when unchanged)
            lib = h.lib
            if mf is None:
                need = _check_size(lib.gast_eval_backward_workspace_bytes(h.h, B, T, ctx.sn),
                                   'gast_eval_backward_workspace_bytes')
                entry, plan = 'gast_eval_backward', ()
            else:
                need = _check_size(lib.gast_chunked_workspace_bytes(h.h, B, T, ctx.sn, mf, 1),
                                   'gast_chunked_workspace_bytes')
                entry, plan = 'gast_eval_backward_chunked', (mf,)
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            dx = torch.empty_like(x) if need_x else None
            views = _bind_grad_views(h, ctx.names, params, False, dev) if need_p else None
            _check(getattr(lib, entry)(h.h, _p(x), _p(dy), _p(dx), 1 if need_p else 0, B, T, ctx.sn, *plan, _p(ws),
                                       ws.numel(), C.c_void_p(st)), entry)
        return (None, None, dx, None, None, None) + (tuple(views) if views is not None else (None,) * ctx.n)


def _no_train(module, what):
    if module.training:
        raise GastError('%s: the training-mode forward/backward exists for the whole model only '
                        '(SpatioTemporalModel / SpatioTemporalModelOptimized1f, what main.train() drives); a sub-module '
                        'on its own runs in eval mode -- call .eval() (there is no silent fallback)' % what)


# ------------------------------------------------------------------------------------------
def model_handle(module, dev):
    """the C handle of a SpatioTemporalModel / ...Optimized1f instance on `dev` (created on first use)"""
    blk0 = module.layers_graph_conv[0].local_graph_layer

    def make():
        return _Handle(module, L.KIND_MODEL, dev, dict(
            num_joints=module.num_joints_in, in_features=module.in_features,
            channels=module._gast_channels, filter_widths=list(module.filter_widths),
            causal=module._gast_causal, dense=module._gast_dense, strided=module._gast_strided, heads=4),
            sym=blk0.gcn_sym.m, con=blk0.gcn_con.m)
    return _handle_for(module, dev, make)


def _strided_now(module, T):
    """1 when the strided schedule runs: always for Optimized1f, and for a dilated model fed exactly one receptive
    field, which computes only what the strided schedule computes (same arithmetic per output), so the unused
    positions are skipped"""
    return 1 if (module._gast_strided or (T == module.receptive_field() and not module._gast_dense)) else 0


def run_model(module, x):
    """SpatioTemporalModelBase.forward (gast_net.py:84-104) on the CUDA library."""
    x = _cuda_input(x, model_dtype(module, 'SpatioTemporalModel.forward'), 'SpatioTemporalModel.forward')
    h = model_handle(module, x.device)
    if module.training:
        refuse_half(module, 'SpatioTemporalModel.forward in train mode', 'training')
        _fp32_only(module, 'SpatioTemporalModel.forward in train mode')
        # both of the reference's training models: Optimized1f (main.py:166-170) and, with
        # --disable-optimizations / stride > 1, the dilated SpatioTemporalModel (main.py:171-175)
        np_ = named_params(module)
        y = _TrainFn.apply(module, h, x, [k for k, _ in np_], *[p for _, p in np_])
    else:
        y = _run_eval(module, h, x, None, 'SpatioTemporalModel.forward')
    module.__dict__['_gast_last_launches'] = h.launches()
    return y


def _run_eval(module, h, x, max_frames, what):
    """the eval-mode forward of x, whole (max_frames None) or in passes (_chunked_forward); with a backward (_EvalFn)
    when autograd is on and x or a parameter requires grad, where the reference's output would carry a grad_fn"""
    strided_now = _strided_now(module, int(x.shape[1]))
    np_ = named_params(module) if torch.is_grad_enabled() else []
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for _, p in np_)):
        refuse_half(module, '%s with autograd (requires_grad input or parameters)' % what, 'gradients')
        _fp32_only(module, '%s with autograd (requires_grad input or parameters)' % what)
        return _EvalFn.apply(module, h, x, strided_now, max_frames, [k for k, _ in np_], *[p for _, p in np_])
    return _chunked_forward(module, h, x, strided_now, max_frames)


def _eval_forward(module, h, x, strided_now, target=None):
    """the eval-mode forward (gast_forward) of x (B,T,J,F) -> y (B,T_out,J,3); with a target of y's shape it returns
    (y, loss), loss the mpjpe of y against it as a 0-d tensor (gast_forward_mpjpe)"""
    dev = x.device
    B, T = int(x.shape[0]), int(x.shape[1])
    with torch.cuda.device(dev):
        st = _stream(dev)
        h.refresh(module, st)
        y = _new_output(module, h, B, T, strided_now, dev, x.dtype)
        if target is None:
            h.forward(x, y, B, T, strided_now, st)
            return y
        if target.shape != y.shape or target.device != dev:
            raise GastError('run_model_mpjpe: target must be %s on %s (got %s on %s)'
                            % (tuple(y.shape), dev, tuple(target.shape), target.device))
        loss = torch.empty((), dtype=torch.float32, device=dev)
        h.forward(x, y, B, T, strided_now, st, target, loss)
    return y, loss


def _new_output(module, h, B, T, strided_now, dev, dtype=torch.float32):
    """an empty (B, T_out, J, 3) model output of `dtype` for an input of T frames on the schedule `strided_now`"""
    T_out = h.lib.gast_out_frames(h.h, T, strided_now)
    if T_out <= 0:
        raise GastError('forward: %s' % L.last_error())
    return torch.empty((B, T_out, module.num_joints_in, 3), dtype=dtype, device=dev)


def run_model_mpjpe(module, x, target):
    """`predicted = model(x); error = mpjpe(predicted, target)` (main.py:270-300, common/loss.py:5-11) as ONE library
    call: the loss is taken in the shrink kernel's epilogue.  Eval mode; returns (predicted, loss) with loss a 0-d
    CUDA tensor.  (The training loss goes through gast_b200.pipeline.mpjpe, which also produces the gradient.)"""
    refuse_half(module, 'run_model_mpjpe', 'the fused mpjpe')
    x = _cuda_f32(x, 'run_model_mpjpe')
    target = _cuda_f32(target, 'run_model_mpjpe (target)')
    _no_train(module, 'run_model_mpjpe')
    h = model_handle(module, x.device)
    y, loss = _eval_forward(module, h, x, _strided_now(module, int(x.shape[1])), target)
    module.__dict__['_gast_last_launches'] = h.launches()
    return y, loss


def run_model_chunked(module, x, max_frames):
    """`model(x)` of a whole model in eval() mode in bounded memory: the library covers the (clip, output frame) grid
    in passes of at most `max_frames` output positions (whole clips, or windows of one clip's output frames with the
    input frames they read), so the workspace depends on max_frames and the architecture, not on the batch or the
    recording length.  Under no_grad, or when neither x nor a parameter requires grad, it is the chunked forward,
    bitwise model(x).  Otherwise the output carries a backward that runs gast_eval_backward_chunked: the gradients of
    model(x)'s backward up to summation order across passes (the same kernels in the same order when one pass covers
    the call).  Train mode
    raises: batch statistics span the whole batch and cannot be chunked."""
    x = _cuda_input(x, model_dtype(module, 'run_model_chunked'), 'run_model_chunked')
    if module.training:
        raise GastError('run_model_chunked: the model is in train mode, whose BatchNorm statistics span the whole '
                        'batch and cannot be chunked; call .eval()')
    h = model_handle(module, x.device)
    y = _run_eval(module, h, x, int(max_frames), 'run_model_chunked')
    module.__dict__['_gast_last_launches'] = h.launches()
    return y


def _chunked_forward(module, h, x, strided_now, max_frames):
    """gast_forward_chunked of x (B,T,J,F) -> y (B,T_out,J,3) on a workspace of its own; max_frames None is the whole
    call, gast_forward (_eval_forward)"""
    if max_frames is None:
        return _eval_forward(module, h, x, strided_now)
    dev = x.device
    B, T = int(x.shape[0]), int(x.shape[1])
    with torch.cuda.device(dev):
        st = _stream(dev)
        h.refresh(module, st)
        y = _new_output(module, h, B, T, strided_now, dev, x.dtype)
        need = _check_size(h.lib.gast_chunked_workspace_bytes(h.h, B, T, strided_now, max_frames, 0),
                           'gast_chunked_workspace_bytes')
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        _check(h.lib.gast_forward_chunked(h.h, _p(x), _p(y), B, T, strided_now, max_frames, _p(ws), ws.numel(),
                                          C.c_void_p(st)), 'gast_forward_chunked')
    return y


def _run_module(module, x, what, kind, cfg, width_out, masks=None, train_ok=False):
    """The forward of a sub-module on its own, channels-last: x (..., J, C) -> (..., J, width_out), all leading rows in
    one library call.  Only a sub-module without BatchNorm or dropout (train_ok) also runs in train mode."""
    refuse_half(module, what, 'a sub-module on its own (only the whole model runs in half)')
    x = _cuda_f32(x, what)
    if not train_ok:
        _no_train(module, what)
    dev = x.device
    *lead, N, Cc = x.shape
    h = _handle_for(module, dev, lambda: _Handle(module, kind, dev, dict(num_joints=N, channels=Cc, **cfg),
                                                 **(masks or {})))
    with torch.cuda.device(dev):
        st = _stream(dev)
        h.refresh(module, st)
        y = torch.empty((*lead, N, width_out), dtype=torch.float32, device=dev)
        h.forward(x, y, math.prod(lead), 1, 0, st)
    return y


def run_block(module, x):
    """GraphAttentionBlock.forward: x (B,C,T,N) -> (B,2C,T,N) (gast_net.py:22-33)."""
    lg = module.local_graph_layer
    return _run_module(module, x.permute(0, 2, 3, 1), 'GraphAttentionBlock.forward', L.KIND_BLOCK, dict(heads=4),
                       2 * x.shape[1], dict(sym=lg.gcn_sym.m, con=lg.gcn_con.m)).permute(0, 3, 1, 2)


def run_local(module, x):
    """LocalGraph.forward: (B,T,J,C) -> (B,T,J,C) (local_attention.py:130-151)."""
    return _run_module(module, x, 'LocalGraph.forward', L.KIND_LOCAL, {}, x.shape[-1],
                       dict(sym=module.gcn_sym.m, con=module.gcn_con.m))


def run_semch(module, x):
    """SemCHGraphConv.forward / SemGraphConv.forward: (B,T,J,Cin) -> (B,T,J,Cout)."""
    shared = 1 if module.e.shape[0] == 1 and module.out_features != 1 else 0
    return _run_module(module, x, 'SemCHGraphConv.forward', L.KIND_SEMCH,
                       dict(channels_out=module.out_features, semch_shared_e=shared,
                            semch_bias=1 if module.bias is not None else 0),
                       module.out_features, dict(sym=module.m), train_ok=True)


def run_multi_global(module, x):
    """MultiGlobalGraph.forward: (B,T,J,C) -> (B,T,J,C) (global_attention.py:103-130)."""
    return _run_module(module, x, 'MultiGlobalGraph.forward', L.KIND_MGLOBAL, dict(heads=module.num_non_local),
                       x.shape[-1])


def run_global_head(module, x):
    """GlobalGraph.forward: (B*T, C, N) -> (B*T, Cg, N) (global_attention.py:52-82)."""
    if module.g_channels != module.inter_channels:
        raise GastError('GlobalGraph with inter_channels == in_channels//2 is not on the lifting path')
    return _run_module(module, x.permute(0, 2, 1), 'GlobalGraph.forward', L.KIND_GLOBAL_HEAD,
                       dict(channels_out=module.inter_channels, heads=1), module.g_channels,
                       train_ok=True).permute(0, 2, 1)


LAUNCH_KINDS = ['expand', 'gemm_ffma_plain', 'gemm_ffma_semch', 'gemm_ffma_global', 'rowdot', 'shrink',
                'gemm_tc_plain', 'gemm_tc_semch', 'gemm_tc_global', 'global_mix']


def profile_forward(module, x, reps=5):
    """Per-launch device times of the model forward (CUDA events inside the library, on the
    launching stream).  Returns per-kernel-kind ms per step and the GEMM-family totals."""
    dev = x.device
    with torch.no_grad():
        run_model(module, x)
    h = module.__dict__['_gast_handles'][(dev.type, dev.index)]
    lib = h.lib
    _check(lib.gast_set_timing(h.h, 1), 'gast_set_timing')
    acc = {}
    n_launch = {}
    try:
        for _ in range(reps):
            with torch.no_grad():
                run_model(module, x)
            ms = (C.c_float * 512)()
            kinds = (C.c_int32 * 512)()
            n = lib.gast_get_timings(h.h, 512, ms, kinds)
            if n < 0:
                raise GastError('gast_get_timings failed')
            n_launch = {}
            for i in range(n):
                k = LAUNCH_KINDS[kinds[i]]
                acc[k] = acc.get(k, 0.0) + ms[i]
                n_launch[k] = n_launch.get(k, 0) + 1
    finally:
        lib.gast_set_timing(h.h, 0)
    per = {k: v / reps for k, v in acc.items()}
    # the GEMM family = every fused channel-contraction launch, plus the attention mix where it runs as its own
    # kernel (it is the epilogue of the `g` GEMM in the fused form)
    fam = lambda k: k.startswith('gemm') or k == 'global_mix'
    gemm = sum(v for k, v in per.items() if fam(k))
    ng = sum(v for k, v in n_launch.items() if fam(k))
    tc = int(lib.gast_last_tc_launch_count(h.h))
    # fp32 grade: three fp16 products on scaled operands, as precise as 3xTF32 (gemm_tc.cuh)
    tc_name = ('wgmma-fp16' if model_dtype(module, 'profile_forward') == torch.float16 or get_precision(module) == 'fp16'
               else 'wgmma-1xtf32' if get_precision(module) == 'tf32' else 'wgmma-3xtf32-grade-3xfp16')
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        run_model(module, x)
        e1.record()
    torch.cuda.synchronize(dev)
    B, T = int(x.shape[0]), int(x.shape[1])
    ws_bytes = int(lib.gast_workspace_bytes(h.h, B, T, _strided_now(module, T)))   # one forward's workspace
    return {'per_kernel_ms': per, 'launches': n_launch, 'gemm_ms_per_step': gemm, 'gemm_launches': ng,
            'step_ms': e0.elapsed_time(e1), 'workspace_bytes': ws_bytes,
            'gemm_core': ('%s x%d + ffma x%d + attention-mix x%d'
                          % (tc_name, tc, ng - tc - n_launch.get('global_mix', 0), n_launch.get('global_mix', 0))) if tc else 'ffma-fp32'}
