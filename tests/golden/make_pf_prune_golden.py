"""Generate tests/golden/pf_prune_golden.npz by running the UNMODIFIED reference (stub-imported) on the seeded cases of
pf_prune_cases.py: leaf-row pruning, a .5 median kiss count, and 1, 2 and 32 pickets.

Run where the reference is installed:  python -m tests.golden.make_pf_prune_golden
Only the reference's outputs are committed; the inputs are regenerated from their seeds and pinned by ``input_sha1``.  A case the
reference raises on stores the exception's type name (``raises_type``) and message (``raises``)."""
from __future__ import annotations

import hashlib
import sys
import warnings
import zipfile

import numpy as np

from tests.golden.make_pf_golden import KEYS
from tests.golden.pf_prune_cases import CASES, case_frame
from tests.golden.refrun import reference_pf

OUT = "tests/golden/pf_prune_golden.npz"


def main():
    from oracle.refstub import import_reference

    import_reference()
    from pylinac import picketfence as rpf

    store = {}
    warnings.simplefilter("ignore")
    for name in CASES:
        a, ps, sid, ck, ak = case_frame(name)
        store[f"{name}/input_sha1"] = np.frombuffer(hashlib.sha1(a.tobytes()).digest(), dtype=np.uint8)
        ck = dict(ck)
        if ck.get("mlc") == "HD":
            ck["mlc"] = rpf.MLC.HD_MILLENNIUM
        try:
            ref = reference_pf(a, ps, sid, ck, ak)
        except Exception as e:  # noqa: BLE001 -- the exception is the reference's result for this case
            store[f"{name}/raises_type"] = np.array(type(e).__name__)
            store[f"{name}/raises"] = np.array(str(e))
            print(name, "raises", type(e).__name__, e)
            continue
        for k in KEYS:
            store[f"{name}/{k}"] = np.asarray(ref[k])
        store[f"{name}/max_error_leaf"] = np.array(str(ref["max_error_leaf"]))
        store[f"{name}/failed_leaves"] = np.array([str(x) for x in ref["failed_leaves"]])
        print(name, "ok", ref["number_of_pickets"], ref["n_meas"])
    _savez_reproducible(OUT, store)


def _savez_reproducible(path, arrays):
    """np.savez_compressed with a fixed member timestamp: the same results give a byte-identical file."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(zi, "w", force_zip64=True) as fh:
                np.lib.format.write_array(fh, np.asanyarray(v), allow_pickle=False)


if __name__ == "__main__":
    sys.exit(main())
