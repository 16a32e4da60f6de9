"""Golden outputs of SORT from the UNMODIFIED reference (lib/track/sort.py) with numba's iou and scipy's
linear_sum_assignment, on the detections of tests/sortref.py's scenarios.

filterpy and skimage are not installed, so two stand-ins go into sys.modules before the import:
- filterpy.kalman.KalmanFilter is tests/sortref.py's KalmanFilter: filterpy 1.4.5's defaults and equations as SORT
  calls them (predict x = Fx, P = F P F' + Q; update with np.linalg.inv and the Joseph form).  It was NOT checked
  against filterpy itself.
- skimage.io is an empty module (Sort does not use it).

Run in the build container only (the GPU box has no reference checkout):
    python tests/golden/make_golden_sort.py
Writes tests/golden/sort.npz (and nothing else).  The detections are not stored: tests/sortref.py's integer formulas
(scenarios) make them.  For each scenario: counts (K,) the rows each update returned, rows (sum, 5) float64 in order;
a scenario where the reference raises stops there and meta records the frame and the exception.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
sys.path.insert(0, os.path.join(HERE, '..'))
import sortref as R                                                   # noqa: E402

filterpy = types.ModuleType('filterpy')
kalman = types.ModuleType('filterpy.kalman')
kalman.KalmanFilter = R.KalmanFilter
filterpy.kalman = kalman
skimage = types.ModuleType('skimage')
skimage.io = types.ModuleType('skimage.io')
sys.modules.update({'filterpy': filterpy, 'filterpy.kalman': kalman, 'skimage': skimage, 'skimage.io': skimage.io})

sys.path.insert(0, os.path.join(REF, 'lib', 'track'))
import sort as _S                                                     # noqa: E402
assert _S.__file__.startswith(REF), _S.__file__


def main():
    import numba
    import scipy
    out, meta = {}, {}
    for name, (max_age, min_hits, frames) in R.scenarios().items():
        _S.KalmanBoxTracker.count = 0
        tracker = _S.Sort(max_age=max_age, min_hits=min_hits)
        counts, rows, raised = [], [], None
        for t, dets in enumerate(frames):
            try:
                r = tracker.update(dets)
            except Exception as e:                  # noqa: BLE001 -- the scenario records what the reference raises
                raised = dict(frame=t, error=type(e).__name__, message=str(e))
                break
            assert r.dtype == np.float64 and r.shape[1] == 5
            counts.append(r.shape[0])
            rows.append(r)
        out['%s_counts' % name] = np.array(counts, np.int32)
        out['%s_rows' % name] = np.concatenate(rows) if rows else np.empty((0, 5))
        meta[name] = dict(max_age=max_age, min_hits=min_hits, frames=len(frames), raised=raised)
        print(name, len(frames), 'frames,', int(np.sum(counts)), 'rows', '' if raised is None else raised)
    out['meta'] = np.array(json.dumps(dict(scenarios=meta, numpy=np.__version__, scipy=scipy.__version__,
                                           numba=numba.__version__)))
    path = os.path.join(HERE, 'sort.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
