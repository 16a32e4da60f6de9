"""Golden outputs of the person detector's letterbox and post-processing from the UNMODIFIED reference
(lib/detector/yolov3/preprocess.py: prep_image; lib/detector/yolov3/util.py: write_results;
lib/detector/yolov3/human_detector.py: yolo_human_det driven by a stand-in model that returns fixed predictions),
with cv2 4.13 (IPP on and off) and torch 2.11 on the CPU.

Run in the build container only (the GPU box has no reference checkout and may have no cv2):
    python tests/golden/make_golden_detection.py
Writes tests/golden/detection.npz (and nothing else).  Frames and predictions are not stored: they are made by the
integer formulas of tests/detectionref.py (synth_frames, prediction_sets).  prep_image's float32 output is stored as
the uint8 it divides (checked to give the reference's floats back exactly), with IPP off; with IPP on as its int8
difference from that.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference'
YOLO = os.path.join(REF, 'lib', 'detector', 'yolov3')

sys.path.insert(0, YOLO)
sys.path.insert(1, os.path.join(REPO, 'tests'))
sys.argv = sys.argv[:1]                 # yolo_human_det parses sys.argv for --nms-thresh

import cv2                                                          # noqa: E402
import preprocess as _P                                             # noqa: E402
import util as _U                                                   # noqa: E402
import human_detector as _H                                         # noqa: E402
import detectionref as R                                            # noqa: E402
assert all(m.__file__.startswith(REF) for m in (_P, _U, _H)), (_P.__file__, _U.__file__, _H.__file__)

D = 416
SIZES = [(1920, 1080), (1080, 1920), (641, 481), (320, 240), (7, 5)]     # (W, H)
CONF = 0.7


def prep(frame):
    img, _, dim = _P.prep_image(frame, D)
    x = img.numpy()[0]
    u8 = np.rint(x * 255).astype(np.uint8)
    assert np.array_equal((u8.astype(np.float32) / np.float32(255)).view(np.uint32), x.view(np.uint32))
    return u8


def human_det(p, D, nms, W, H):
    sys.argv = [sys.argv[0], '--nms-thresh', repr(nms)]
    model = lambda img, cuda: torch.from_numpy(p.copy())[None]       # noqa: E731
    return _H.yolo_human_det(np.zeros((H, W, 3), np.uint8), model, reso=D, confidence=CONF)


def main():
    out = {}
    for k, (W, H) in enumerate(SIZES):
        frame = R.synth_frames(1, H, W, seed=k)[0]
        cv2.ipp.setUseIPP(False)
        off = prep(frame)
        cv2.ipp.setUseIPP(True)
        on = prep(frame)
        out['prep_off_%d' % k] = off
        out['prep_ipp_diff_%d' % k] = (on.astype(np.int16) - off).astype(np.int8)
    cv2.ipp.setUseIPP(False)

    sets = R.prediction_sets()
    meta_sets = {}
    for name, (d, p, nms, (W, H)) in sets.items():
        b, s = human_det(p, d, nms, W, H)
        meta_sets[name] = dict(D=d, nms=nms, W=W, H=H, n=0 if b is None else int(b.shape[0]))
        if b is not None:
            assert b.dtype == np.float32 and s.dtype == np.float32
            out['det_%s_boxes' % name], out['det_%s_scores' % name] = b, s
    sys.argv = sys.argv[:1]

    # write_results on a batch: both images with persons, then the early return at an image without one
    batches = {'wr_two': ['iou_edge', 'clamp'], 'wr_early': ['clamp', 'none', 'single']}
    for key, names in batches.items():
        pred = torch.from_numpy(np.stack([sets[n][1] for n in names]))
        with torch.no_grad():
            r = _U.write_results(pred.clone(), CONF, 80, nms=True, nms_conf=0.4, det_hm=True)
        out[key] = r.numpy()

    meta = dict(D=D, sizes=SIZES, conf=CONF, sets=meta_sets, batches=batches, cv2=cv2.__version__,
                torch=torch.__version__, numpy=np.__version__)
    out['meta'] = np.array(json.dumps(meta))
    path = os.path.join(HERE, 'detection.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
