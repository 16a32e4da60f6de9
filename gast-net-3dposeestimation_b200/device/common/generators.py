"""Device-side counterpart of the reference's common/generators.py: batches assembled ON THE DEVICE
(import as device.common.generators: it yields CUDA tensors where the reference yields numpy arrays, so it
does not shadow the reference module).

`ChunkedGenerator` (generators.py:4-157) keeps the reference's constructor, pair list, shuffling
(`np.random.RandomState(seed).permutation`, so the batch order is the reference's) and `next_epoch`
protocol, but the sequences live concatenated in HBM (gast_b200.pipeline.DeviceSequences) and each batch
is one gather kernel (edge padding, horizontal flip, left/right swap: csrc/pipeline.cuh) that yields CUDA
float32 tensors -- the reference fills float64 numpy buffers chunk by chunk in a Python loop and the
training loop then casts and uploads them (main.py:219-223).  `UnchunkedGenerator` (generators.py:160-235)
yields one padded (and, with augment, mirrored) sequence at a time, also as CUDA tensors.  Both take the
sequences as numpy arrays or as CUDA tensors (gast_b200.dataset's fetch), the latter without a host round trip.
"""
from itertools import zip_longest

import numpy as np
import torch

from gast_b200 import pipeline as _P
from gast_b200 import tta as _T


class ChunkedGenerator(object):
    def __init__(self, batch_size, cameras, poses_3d, poses_2d, chunk_length, pad=0, causal_shift=0, shuffle=True,
                 random_seed=1234, augment=False, kps_left=None, kps_right=None, joints_left=None, joints_right=None,
                 endless=False, device='cuda'):
        assert poses_3d is None or len(poses_3d) == len(poses_2d), (len(poses_3d), len(poses_2d))
        assert cameras is None or len(cameras) == len(poses_2d)
        pairs = []                                     # (seq_idx, start_frame, end_frame, flip), generators.py:31-41
        for i in range(len(poses_2d)):
            assert poses_3d is None or poses_3d[i].shape[0] == poses_2d[i].shape[0]
            n_chunks = (poses_2d[i].shape[0] + chunk_length - 1) // chunk_length
            offset = (n_chunks * chunk_length - poses_2d[i].shape[0]) // 2
            bounds = np.arange(n_chunks + 1) * chunk_length - offset
            for flip in ((0, 1) if augment else (0,)):
                blk = np.stack([np.full(n_chunks, i), bounds[:-1], bounds[1:], np.full(n_chunks, flip)], axis=1)
                pairs.append(blk.astype(np.int64))
        self.pairs = np.concatenate(pairs, axis=0) if pairs else np.zeros((0, 4), np.int64)
        self.num_batches = (len(self.pairs) + batch_size - 1) // batch_size
        self.batch_size = batch_size
        self.random = np.random.RandomState(random_seed)
        self.shuffle = shuffle
        self.pad = pad
        self.causal_shift = causal_shift
        self.endless = endless
        self.state = None
        self.chunk_length = chunk_length
        self.seqs = _P.DeviceSequences(poses_2d, poses_3d, cameras, device=device)
        self.cameras = cameras
        self.poses_3d = poses_3d
        self.poses_2d = poses_2d
        self.augment = augment
        self.kps_left = kps_left
        self.kps_right = kps_right
        self.joints_left = joints_left
        self.joints_right = joints_right

    def num_frames(self):
        return self.num_batches * self.batch_size

    def random_state(self):
        return self.random

    def set_random_state(self, random):
        self.random = random

    def augment_enabled(self):
        return self.augment

    def next_pairs(self):
        if self.state is None:
            pairs = self.random.permutation(self.pairs) if self.shuffle else self.pairs
            return 0, pairs
        return self.state

    def next_epoch(self):
        enabled = True
        while enabled:
            start_idx, pairs = self.next_pairs()
            for b_i in range(start_idx, self.num_batches):
                chunks = pairs[b_i * self.batch_size:(b_i + 1) * self.batch_size]
                cam, b3, b2 = _P.chunk_gather(self.seqs, chunks, self.chunk_length, self.pad, self.causal_shift,
                                              self.kps_left, self.kps_right, self.joints_left, self.joints_right)
                if self.endless:
                    self.state = (b_i + 1, pairs)
                yield cam, b3, b2
            if self.endless:
                self.state = None
            else:
                enabled = False


class UnchunkedGenerator(object):
    def __init__(self, cameras, poses_3d, poses_2d, pad=0, causal_shift=0, augment=False, kps_left=None, kps_right=None,
                 joints_left=None, joints_right=None, device='cuda'):
        assert poses_3d is None or len(poses_3d) == len(poses_2d)
        assert cameras is None or len(cameras) == len(poses_2d)
        self.augment = augment
        self.kps_left = kps_left
        self.kps_right = kps_right
        self.joints_left = joints_left
        self.joints_right = joints_right
        self.pad = pad
        self.causal_shift = causal_shift
        self.cameras = [] if cameras is None else cameras
        self.poses_3d = [] if poses_3d is None else poses_3d
        self.poses_2d = poses_2d
        self.device = device

    def num_frames(self):
        return sum(p.shape[0] for p in self.poses_2d)

    def augment_enabled(self):
        return self.augment

    def set_augment(self, augment):
        self.augment = augment

    def _dev(self, a):
        if isinstance(a, torch.Tensor) and a.is_cuda:                 # fetched on the device: no host round trip
            return a.to(device=self.device, dtype=torch.float32).contiguous()
        return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(self.device)

    def next_epoch(self):
        for seq_cam, seq_3d, seq_2d in zip_longest(self.cameras, self.poses_3d, self.poses_2d):
            both = _T.tta_prepare(self._dev(seq_2d), self.pad, self.causal_shift,
                                  self.kps_left if self.augment else [], self.kps_right if self.augment else [])
            batch_2d = both if self.augment else both[:1]
            batch_cam = batch_3d = None
            if seq_cam is not None:
                batch_cam = self._dev(seq_cam)[None]
                if self.augment:
                    batch_cam = torch.cat((batch_cam, batch_cam), 0)
                    batch_cam[1, 2] *= -1
                    batch_cam[1, 7] *= -1
            if seq_3d is not None:
                s3 = self._dev(seq_3d)
                if self.augment:
                    batch_3d = _T.tta_prepare(s3, 0, 0, self.joints_left, self.joints_right)
                else:
                    batch_3d = s3[None]
            yield batch_cam, batch_3d, batch_2d
