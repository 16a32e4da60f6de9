"""The reference's main.train (oracle/_ref/main.py, staged by build()) driven by the DEVICE ChunkedGenerator.

main.train turns each batch into a CUDA tensor with `torch.from_numpy(batch.astype('float32'))` and `.cuda()`
(main.py:219-223).  The device generator's batches already are CUDA float32 tensors, so `main_train_device` runs
main.train's own code object with those two conversions as identities: every other line -- zero_grad, the forward,
the loss, the backward, the optimiser step and the loss bookkeeping -- is the reference's, unchanged.  INTEGRATION.md
§3 makes the same edit by deleting the lines.
"""
import types

import torch


class _CudaBatch(object):
    """a CUDA batch whose `.astype('float32')` is the batch itself"""

    def __init__(self, t):
        self.t = t

    def astype(self, dtype):
        assert dtype == 'float32' and self.t.dtype == torch.float32
        return self.t


class _DeviceBatches(object):
    def __init__(self, gen):
        self.gen = gen

    def next_epoch(self):
        for cam, b3, b2 in self.gen.next_epoch():
            yield cam, _CudaBatch(b3), _CudaBatch(b2)


def main_train_device(main, model, gen, optimizer):
    """main.train(model, gen, optimizer) over the device generator `gen`"""
    g = dict(main.train.__globals__)
    g['torch'] = types.SimpleNamespace(from_numpy=lambda a: a, cuda=torch.cuda)
    fn = types.FunctionType(main.train.__code__, g, 'train')
    return fn(model, _DeviceBatches(gen), optimizer)
