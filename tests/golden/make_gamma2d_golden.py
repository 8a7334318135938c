"""Generate tests/golden/gamma2d_golden.npz: pylinac.core.gamma.gamma_2d of the UNMODIFIED reference (core/gamma.py:229-330,
stub-imported) on the pairs of gamma2d_cases.py, and the exceptions of its ERROR_CASES.  skimage is stubbed at import time, so the
module's ``disk`` is rebound to the restated one (oracle/skimage_draw.py).  Run here:  python -m tests.golden.make_gamma2d_golden"""
from __future__ import annotations

import sys
import warnings

import numpy as np

from tests.golden.gamma2d_cases import CASES, ERROR_CASES, case_pair


def main():
    from oracle import skimage_draw
    from oracle.refstub import import_reference

    import_reference()
    import pylinac.core.gamma as rgamma

    rgamma.disk = skimage_draw.disk
    store = {}
    warnings.simplefilter("ignore")
    for name in CASES:
        ref, ev, kw = case_pair(name)
        g = rgamma.gamma_2d(ref, ev, **kw)
        store[name] = np.asarray(g)
        print(name, g.dtype, g.shape, float(np.nanmax(g)) if np.isfinite(g).any() else None, int(np.isnan(g).sum()))
    for name, (rshape, eshape, kw) in ERROR_CASES.items():
        try:
            rgamma.gamma_2d(np.ones(rshape), np.ones(eshape), **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the golden
            store["error:" + name] = np.array([type(e).__name__, str(e)])
            print(name, type(e).__name__, repr(str(e)))
        else:
            raise AssertionError(f"{name}: the reference raised nothing")
    np.savez_compressed("tests/golden/gamma2d_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
