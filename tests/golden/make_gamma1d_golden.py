"""Generate tests/golden/gamma1d_golden.npz: pylinac.core.gamma.gamma_geometric / gamma_1d and the profile gamma methods of the
UNMODIFIED reference (stub-imported) on the cases of gamma1d_cases.py, and the exceptions of its ERROR_CASES.
Run here:  python -m tests.golden.make_gamma1d_golden"""
from __future__ import annotations

import sys
import warnings

import numpy as np

from tests.golden.gamma1d_cases import CASES, ERROR_CASES, PROFILE_CASES, case_args, error_args, profile_signal


def _store_error(store, key, call):
    try:
        call()
    except Exception as e:  # noqa: BLE001 -- the exception is the golden
        store["error:" + key] = np.array([type(e).__name__, str(e)])
        print(key, type(e).__name__, repr(str(e)))
        return True
    return False


def main():
    from oracle.refstub import import_reference

    import_reference()
    import pylinac.core.gamma as rgamma
    import pylinac.core.profile as rprofile

    funcs = {"geometric": rgamma.gamma_geometric, "1d": rgamma.gamma_1d}
    store = {}
    warnings.simplefilter("ignore")
    for name in CASES:
        fn, ref, ev, rc, ec, kw = case_args(name)
        out = {}
        if _store_error(store, name, lambda: out.setdefault("r", funcs[fn](ref, ev, rc, ec, **kw))):
            continue
        r = out["r"]
        if fn == "1d":
            store[name], store[name + ":samples"], store[name + ":x"] = r
        else:
            store[name] = r
        g = store[name]
        print(name, g.dtype, g.shape, int(np.isnan(g.astype(float)).sum()))
    for name in ERROR_CASES:
        fn, ref, ev, rc, ec, kw = error_args(name)
        if not _store_error(store, name, lambda: funcs[fn](ref, ev, rc, ec, **kw)):
            raise AssertionError(f"{name}: the reference raised nothing")
    for name, (method, nr, dr, ne, de, kw) in PROFILE_CASES.items():
        rng = np.random.default_rng(4000 + sorted(PROFILE_CASES).index(name))
        a, b = profile_signal(nr, rng), profile_signal(ne, rng, centre=0.8)
        if method == "physical":
            ra, rb = rprofile.FWXMProfilePhysical(a, dpmm=dr), rprofile.FWXMProfilePhysical(b, dpmm=de)
            r = ra.gamma(rb, **kw)
            if kw.get("return_profiles"):
                r, pa, pb = r
                for tag, p in (("ref", pa), ("eval", pb)):
                    store[f"{name}:{tag}:values"] = np.asarray(p.values)
                    store[f"{name}:{tag}:x_values"] = np.asarray(p.x_values)
                    store[f"{name}:{tag}:physical_x_values"] = np.asarray(p.physical_x_values)
        else:
            ra, rb = rprofile.SingleProfile(a, dpmm=dr), rprofile.SingleProfile(b, dpmm=de)
            r = ra.gamma(rb, **kw)
        store[name] = np.asarray(r)
        print(name, r.shape, int(np.isnan(r).sum()))
    a = profile_signal(101, np.random.default_rng(4100))
    if not _store_error(store, "single_profile_no_dpmm",
                        lambda: rprofile.SingleProfile(a, dpmm=None).gamma(rprofile.SingleProfile(a, dpmm=2.0))):
        raise AssertionError("single_profile_no_dpmm: the reference raised nothing")
    np.savez_compressed("tests/golden/gamma1d_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
