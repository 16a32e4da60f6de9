"""Whole training epochs on the device: trainval.py's loop (trainval.py:113-165 -> main.train, main.py:213-243, and
main.eval, main.py:246-296) with one CUDA-graph replay per batch and one host synchronisation per epoch.

A step is the batch gather (gast_chunk_gather_indexed), the root zeroing of the target (main.py:225), the training
forward, the loss (common/loss.py:5-11, torch's ops as main.train runs them), the backward into one flat gradient
buffer, the Adam(amsgrad) step (gast_adam_step_indexed) and the loss bookkeeping (gast_epoch_loss_accumulate).  Every
per-step value -- which pairs to gather, Adam's step size and bias correction, where the loss goes -- is read on the
device from the epoch's batch counter, so the step is captured once per batch shape and replayed for every batch.
Batch order, arithmetic and results are main.train's (DESIGN.md §8.3).
"""
import copy

import numpy as np
import torch

from . import engine as _E
from . import pipeline as _P
from .dist import FlatGradBuffer
from .engine import GastError
from .evaluation import evaluate_sequences
from .trainer import mpjpe


def _pinned(a):
    """a host numpy array as a page-locked tensor: uploaded with copy_(non_blocking=True), no host wait"""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


class EpochTrainer(object):
    """Runs trainval.py's epochs for `model_pos_train` (SpatioTemporalModelOptimized1f at chunk length 1, or the
    dilated SpatioTemporalModel, in train mode) over `train_generator` (a device.common.generators.ChunkedGenerator,
    not endless, with 3D poses) with `optimizer` (a pipeline.FusedAdam over exactly the model's trainable parameters).

    train_epoch() returns main.train(model_pos_train, train_generator, optimizer)'s value bit for bit; the parameters,
    BatchNorm statistics, Adam moments and optimizer.step_count end where main.train leaves them.  Each epoch permutes
    the pairs with the generator's own RandomState (as its next_epoch does) and reads the lr from
    optimizer.param_groups[0]['lr'], so trainval's `param_group['lr'] *= lr_decay` keeps working; betas, eps,
    weight_decay and amsgrad are fixed at construction, as are the GEMM core and the precisions.

    Construction captures the step for the full batch and, when the pair count is not a multiple of the batch size,
    for the shorter last batch, after one warm-up of each on a side stream.  It leaves every parameter, BatchNorm
    buffer, Adam moment, step_count and the dropout counter as it found them.  The parameters' .grad become views of
    the trainer's flat gradient buffer.  Dropout takes its masks from the model's device dropout counter
    (`_gast_dropout_state`, created at 0 when absent), which advances once per batch."""

    def __init__(self, model_pos_train, train_generator, optimizer, checkpoint=None):
        from device.common.generators import ChunkedGenerator
        m, gen, opt = model_pos_train, train_generator, optimizer
        if not hasattr(m, 'layers_graph_conv') or not hasattr(m, 'receptive_field'):
            raise GastError('EpochTrainer: the model must be a SpatioTemporalModel or SpatioTemporalModelOptimized1f '
                            '(got %s)' % type(m).__name__)
        _E.refuse_half(m, 'EpochTrainer', 'training')
        _E._fp32_only(m, 'EpochTrainer')
        if not m.training:
            raise GastError('EpochTrainer: the model is in eval mode; call model.train() (main.train trains it in '
                            'train mode, trainval.py:117)')
        if torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            raise GastError('EpochTrainer: one process, one GPU; with torch.distributed at world size %d use '
                            'gast_b200.trainer.DataParallelTrainer' % torch.distributed.get_world_size())
        trainable = [p for p in m.parameters() if p.requires_grad]
        if not isinstance(opt, _P.FusedAdam) or len(opt.params) != len(trainable) \
                or {id(p) for p in opt.params} != {id(p) for p in trainable}:
            raise GastError('EpochTrainer: the optimizer must be a gast_b200.pipeline.FusedAdam over exactly the '
                            "model's trainable parameters (got %s)" % type(opt).__name__)
        if not isinstance(gen, ChunkedGenerator) or gen.endless or gen.poses_3d is None or len(gen.pairs) == 0:
            raise GastError('EpochTrainer: the generator must be a device.common.generators.ChunkedGenerator with 3D '
                            'poses, at least one pair, and not endless')
        if m.receptive_field() != 2 * gen.pad + 1 or (m._gast_strided and gen.chunk_length != 1):
            raise GastError('EpochTrainer: the generator pads %d frames per side at chunk length %d; the model needs '
                            'pad = %d%s' % (gen.pad, gen.chunk_length, (m.receptive_field() - 1) // 2,
                                            ' and chunk length 1 (SpatioTemporalModelOptimized1f)'
                                            if m._gast_strided else ''))
        self.model, self.gen, self.opt = m, gen, opt
        dev = trainable[0].device
        self.B = int(gen.batch_size)
        self.n_pairs = len(gen.pairs)
        self.n_batches = int(gen.num_batches)
        self.tail = self.n_pairs - (self.n_batches - 1) * self.B
        self.frames = self.n_pairs * int(gen.chunk_length)        # main.train's N
        g = opt.param_groups[0]
        self._fixed = (tuple(g['betas']), g['eps'], g['weight_decay'], g['amsgrad'])
        self.pairs = torch.empty((self.n_pairs, 4), dtype=torch.int32, device=dev)
        self.coef = torch.empty((self.n_batches, 2), dtype=torch.float32, device=dev)
        self.batch = torch.zeros((), dtype=torch.int64, device=dev)
        self.loss_sum = torch.zeros((), dtype=torch.float64, device=dev)
        self.losses = torch.zeros((self.n_batches,), dtype=torch.float32, device=dev)
        self.flat = FlatGradBuffer(m.parameters())
        if m.__dict__.get('_gast_dropout_state') is None:
            m.__dict__['_gast_dropout_state'] = torch.zeros(1, dtype=torch.int64, device=dev)
        self.epoch = 0
        self.graphs = {}
        self._capture(dev)
        if checkpoint is not None:
            self.load_checkpoint(checkpoint)

    # ---------------------------------------------------------------------------------------------------------------
    def _state(self):
        """every tensor a step writes besides its scratch: parameters, BatchNorm buffers, Adam moments, the dropout
        and batch counters and the epoch's loss records"""
        o = self.opt
        return ([v for _, v in _E.named_tensors(self.model)] + [o.exp_avg, o.exp_avg_sq]
                + ([o.max_exp_avg_sq] if o.max_exp_avg_sq is not None else [])
                + [self.model.__dict__['_gast_dropout_state'], self.batch, self.loss_sum, self.losses])

    def _step(self, B):
        gen = self.gen
        _, b3, b2 = _P.chunk_gather_indexed(gen.seqs, self.pairs, self.batch, B, self.B, gen.chunk_length, gen.pad,
                                            gen.causal_shift, gen.kps_left, gen.kps_right, gen.joints_left,
                                            gen.joints_right)
        b3[:, :, 0] = 0                                           # main.py:225
        self.flat.zero_()
        loss = mpjpe(self.model(b2), b3)
        loss.backward()
        self.opt.step_indexed(self.coef, self.batch)
        _P.epoch_loss_accumulate(loss.detach(), B * int(b3.shape[1]), self.loss_sum, self.losses, self.batch)

    def _capture(self, dev):
        """warm up and capture the step of each batch size, then put every tensor of _state() back byte for byte"""
        m = self.model
        shapes = [self.B] + ([self.tail] if self.tail != self.B else [])
        with torch.no_grad():       # a clone with a grad_fn would keep a gradient accumulator made on this stream
            saved = [t.clone() for t in self._state()]
        direct = m.__dict__.get('_gast_direct_grads')
        m.__dict__['_gast_direct_grads'] = True                   # the backward writes straight into self.flat
        self.opt._build_table()                                   # its upload may not happen during the capture
        self.pairs.copy_(torch.as_tensor(self.gen.pairs.astype(np.int32)))   # valid rows for the warm-up steps
        self.coef.copy_(torch.as_tensor(_P.adam_step_table(self.opt.param_groups[0]['lr'], self._fixed[0], 1,
                                                           self.n_batches)))
        try:
            with torch.random.fork_rng(devices=[]):               # the eager dropout seed draw: no trace in torch's RNG
                side = torch.cuda.Stream(dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):                     # allocator, attribute opt-ins, handles: not captured
                    for B in shapes:
                        self.batch.fill_(0 if B == self.B else self.n_batches - 1)
                        self._step(B)
                torch.cuda.current_stream(dev).wait_stream(side)
                pool = None                                       # one memory pool: the graphs never run at once
                for B in shapes:
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, pool=pool):
                        self._step(B)
                    pool = g.pool()
                    self.graphs[B] = g
        finally:                                                  # a capture only records: undo the warm-up steps
            with torch.no_grad():
                for t, s in zip(self._state(), saved):
                    t.copy_(s)
            if direct is None:
                m.__dict__.pop('_gast_direct_grads', None)
            else:
                m.__dict__['_gast_direct_grads'] = direct

    # ---------------------------------------------------------------------------------------------------------------
    def train_epoch_async(self):
        """One epoch without a host synchronisation: returns (the fp64 0-d CUDA sum over the batches of
        B * T_out * loss, the (n_batches,) float32 CUDA per-step losses), both copies of the epoch's records.  The
        epoch loss is the sum over `self.frames`."""
        g = self.opt.param_groups[0]
        if (tuple(g['betas']), g['eps'], g['weight_decay'], g['amsgrad']) != self._fixed:
            raise GastError('EpochTrainer: betas, eps, weight_decay and amsgrad were captured as %r; only the lr may '
                            'change between epochs' % (self._fixed,))
        _, pairs = self.gen.next_pairs()                          # the generator's own permutation (next_epoch)
        self.pairs.copy_(_pinned(pairs.astype(np.int32)), non_blocking=True)
        coef = _P.adam_step_table(g['lr'], self._fixed[0], self.opt.step_count + 1, self.n_batches)
        self.coef.copy_(_pinned(coef), non_blocking=True)
        self.batch.zero_()
        self.loss_sum.zero_()
        full = self.graphs[self.B]
        for _ in range(self.n_batches - 1):
            full.replay()
        self.graphs[self.tail].replay()
        self.opt.step_count += self.n_batches
        # the replays wrote the parameters and buffers behind autograd's back: new versions make the engine's eval-mode
        # constants refresh (as FusedAdam.step and the eager training forward do)
        torch.autograd.graph.increment_version([v for _, v in _E.named_tensors(self.model)])
        self.epoch += 1
        return self.loss_sum.clone(), self.losses.clone()

    def train_epoch(self):
        """main.train(model_pos_train, train_generator, optimizer) for one epoch: the epoch loss as a Python float,
        after one synchronisation"""
        loss_sum, _ = self.train_epoch_async()
        return loss_sum.item() / self.frames

    def eval_epoch(self, model_pos, test_2d, test_3d, train_2d, train_3d):
        """main.eval's (losses_3d_valid_ave, losses_3d_train_eval_ave) (main.py:246-296): model_pos takes the training
        model's state_dict, goes to eval mode, and scores each split (lists of (T,J,F) 2D and (T,J,3) 3D sequences,
        as fetch builds them) with evaluate_sequences, without augmentation, against root-zeroed targets.  Returns
        the frame-weighted mpjpe of each split; zero-length sequences are skipped (main.py:275-277)."""
        model_pos.load_state_dict(self.model.state_dict())
        model_pos.eval()

        def score(p2, p3):
            keep = [i for i in range(len(p2)) if int(p2[i].shape[0]) > 0]
            if not keep:
                return float('nan')
            res = evaluate_sequences(model_pos, [p2[i] for i in keep], [p3[i] for i in keep], augment=False,
                                     procrustes=False, zero_root=True)
            return float(res[None].mpjpe)
        with torch.no_grad():
            return score(test_2d, test_3d), score(train_2d, train_3d)

    # ---------------------------------------------------------------------------------------------------------------
    def checkpoint(self):
        """trainval's checkpoint dict (trainval.py:149-157,171-177) as a snapshot: epoch (the epochs trained), lr,
        random_state (the generator's), optimizer (FusedAdam's state_dict) and model_pos (the model's state_dict)"""
        sd = self.opt.state_dict()
        return {'epoch': self.epoch, 'lr': self.opt.param_groups[0]['lr'],
                'random_state': copy.deepcopy(self.gen.random_state()),
                'optimizer': {k: (v.clone() if isinstance(v, torch.Tensor) else copy.deepcopy(v)) for k, v in sd.items()},
                'model_pos': {k: v.clone() for k, v in self.model.state_dict().items()}}

    def load_checkpoint(self, checkpoint):
        """resume from checkpoint(): the model, the optimizer (lr included), the generator's RandomState and the
        epoch count"""
        self.model.load_state_dict(checkpoint['model_pos'])
        self.opt.load_state_dict(checkpoint['optimizer'])
        self.gen.set_random_state(copy.deepcopy(checkpoint['random_state']))
        self.epoch = int(checkpoint['epoch'])
