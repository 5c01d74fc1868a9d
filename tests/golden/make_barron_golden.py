"""Builds tests/golden/barron_reference_fixtures.npz from the reference's OWN test fixtures (argument: a checkout
of google/neural-light-transport; the tests only read the committed npz):

  * third_party/robust_loss/data/wavelet_golden.mat -- an 83 x 71 RGB image and its 5-level CDF 9/7 pyramid made
    by an independent implementation (see wavelet_test.py:146-172); stored here as float64 arrays
    `image`, `band_<level>_<k>`, `residual`;
  * third_party/robust_loss/data/partition_spline.npz -- only `x_scale` and the two knots around alpha = 1.
"""
import os
import sys

import numpy as np
import scipy.io

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else '.', 'third_party', 'robust_loss', 'data')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'barron_reference_fixtures.npz')


def main():
    mat = scipy.io.loadmat(os.path.join(REF, 'wavelet_golden.mat'))
    out = {'image': np.asarray(mat['I_color'], dtype=np.float64)}
    pyr = mat['pyr_color'][0, :].tolist()
    for level, bands in enumerate(pyr[:-1]):
        for k, band in enumerate(bands.flatten()):
            out['band_%d_%d' % (level, k)] = np.asarray(band, dtype=np.float64)
    out['residual'] = np.asarray(pyr[-1], dtype=np.float64)
    out['num_levels'] = np.int64(len(pyr) - 1)
    with np.load(os.path.join(REF, 'partition_spline.npz')) as f:
        x_scale = int(f['x_scale'])
        x = ((2.25 * 1.0 - 4.5) / (abs(1.0 - 2.0) + 0.25) + 1.0 + 2.0) * x_scale      # alpha = 1
        lo = int(np.floor(x))
        out['spline_x_scale'] = np.int64(x_scale)
        out['spline_knot_lo'] = np.int64(lo)
        out['spline_values'] = f['values'][lo:lo + 2].astype(np.float64)
        out['spline_tangents'] = f['tangents'][lo:lo + 2].astype(np.float64)
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, {k: getattr(v, 'shape', ()) for k, v in out.items()})


if __name__ == '__main__':
    main()
