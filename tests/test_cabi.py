"""CPU: the C-ABI shared library loads and exports every symbol include/epid.h declares, and the ctypes binding's structs and
signatures agree with the header (no compute calls)."""
import ctypes
import os
import re
import subprocess

import numpy as np

from pylinac_b200 import _native as nat

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "epid.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(epid_[a-z0-9_]+)\s*\(", src)))


def test_header_functions_are_exported_and_bound():
    names = declared_functions()
    assert len(names) >= 40
    handle = ctypes.CDLL(nat.LIB_PATH)
    for n in names:
        assert hasattr(handle, n), f"libepid.so does not export {n}"
    bound = set(nat.exported_symbols())
    assert set(names) <= bound, sorted(set(names) - bound)
    assert bound <= set(names), sorted(bound - set(names))


# every struct of the header and its one Python declaration: a ctypes Structure for the params the binding passes by pointer, a numpy
# dtype for the result rows the caller reads
STRUCTS = {
    "epid_peak_params": nat.PeakParams,
    "epid_pf_params": nat.PFParams,
    "epid_pf_summary": nat.PF_SUMMARY_DTYPE,
    "epid_pf_meas": nat.PF_MEAS_DTYPE,
    "epid_star_params": nat.StarParams,
    "epid_star_result": nat.STAR_RESULT_DTYPE,
    "epid_field_params": nat.FieldParams,
    "epid_field_result": nat.FIELD_RESULT_DTYPE,
    "epid_sp_params": nat.SpParams,
    "epid_sp_result": nat.SP_RESULT_DTYPE,
    "epid_wl_params": nat.WlParams,
    "epid_wl_result": nat.WL_RESULT_DTYPE,
    "epid_disk_params": nat.DiskParams,
    "epid_disk_result": nat.DISK_RESULT_DTYPE,
    "epid_vmat_params": nat.VmatParams,
    "epid_vmat_row": nat.VMAT_RESULT_DTYPE,
    "epid_locate_params": nat.LocateParams,
    "epid_region": nat.REGION_DTYPE,
    "epid_lr_params": nat.LrParams,
    "epid_lr_result": nat.LR_RESULT_DTYPE,
}


def header_source():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def python_layout(decl):
    """(size, {member: (offset, size)}) of a ctypes Structure or a numpy dtype"""
    if isinstance(decl, np.dtype):
        return decl.itemsize, {name: (decl.fields[name][1], decl.fields[name][0].itemsize) for name in decl.names}
    return ctypes.sizeof(decl), {name: (getattr(decl, name).offset, getattr(decl, name).size) for name, *_ in decl._fields_}


def test_structs_match_the_header(tmp_path):
    """Size, member offsets and member sizes of every Python declaration, as the host C++ compiler lays out the header's struct."""
    declared = re.findall(r"typedef\s+struct\s*\{[^}]*\}\s*(epid_\w+)\s*;", header_source())
    assert sorted(declared) == sorted(STRUCTS), sorted(set(declared) ^ set(STRUCTS))
    prints = []
    for s, decl in STRUCTS.items():
        prints.append(f'std::printf("{s} sizeof %zu\\n", sizeof({s}));')
        prints += [f'std::printf("{s} {m} %zu %zu\\n", offsetof({s}, {m}), sizeof({s}::{m}));' for m in python_layout(decl)[1]]
    src = tmp_path / "layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "layout")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True, text=True).stdout
    header = {(s, m): tuple(int(v) for v in vals) for s, m, *vals in (line.split() for line in out.splitlines())}
    wrong = []
    for s, decl in STRUCTS.items():
        size, members = python_layout(decl)
        if header[s, "sizeof"] != (size,):
            wrong.append(f"{s}: sizeof {header[s, 'sizeof'][0]} in the header, {size} in the binding")
        wrong += [f"{s}.{m}: (offset, size) {header[s, m]} in the header, {om} in the binding"
                  for m, om in members.items() if header[s, m] != om]
    assert not wrong, "\n".join(wrong)


ARG_KINDS = {"int32_t": "int32", "int64_t": "int64", "size_t": "size_t", "double": "double", "float": "float"}
CTYPES_KINDS = {ctypes.c_int32: "int32", ctypes.c_int64: "int64", ctypes.c_size_t: "size_t", ctypes.c_double: "double",
                ctypes.c_float: "float"}


def header_prototypes():
    """{name: (return type, [argument kind])} of every function the header declares"""
    protos = {}
    for ret, name, args in re.findall(r"^\s*(int32_t|const char\s*\*)\s*(epid_\w+)\s*\(([^)]*)\)\s*;", header_source(), flags=re.M):
        args = [a.split() for a in args.split(",") if a.strip() != "void"]
        protos[name] = (ret, ["pointer" if "*" in "".join(a) else ARG_KINDS[" ".join(a[:-1])] for a in args])
    return protos


def binding_kind(t):
    return "pointer" if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer) else CTYPES_KINDS[t]


def test_signatures_match_the_header():
    """Arity and argument kinds of every ctypes signature, and the return type the binding sets, against the header's prototype."""
    protos = header_prototypes()
    assert sorted(protos) == declared_functions()
    assert protos["epid_last_error"] == ("const char*", [])
    wrong = [f"{name}: {protos[name]} in the header, binding {('int32_t', [binding_kind(t) for t in args])}"
             for name, args in nat._SIGNATURES.items() if protos[name] != ("int32_t", [binding_kind(t) for t in args])]
    assert not wrong, "\n".join(wrong)


def test_no_device_is_reported_not_faked():
    """Without a GPU every compute entry point must fail loudly (EPID_ERR_NO_DEVICE), never fall back to the CPU."""
    import numpy as np
    import pytest

    if nat.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(nat.NoDeviceError):
        nat.Context(0)
    from pylinac_b200 import picketfence as pf

    with pytest.raises(nat.NoDeviceError):
        pf.analyze_batch(np.zeros((1, 64, 64), np.uint16), 2.56)


def test_product_never_imports_the_oracle_and_has_one_scipy_call_site():
    """The oracle is test infrastructure: nothing under pylinac_b200/ may import it (a product path through the oracle would void
    every parity claim).  scipy is allowed in exactly one place: the set-level Winston-Lutz minimisation the reference itself does
    on the host (winston_lutz.py:1614-1640)."""
    import ast
    import pathlib

    root = pathlib.Path(__file__).resolve().parents[1] / "pylinac_b200"
    scipy_sites = []
    for path in root.rglob("*.py"):
        tree = ast.parse(path.read_text())
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom) and node.module:
                names = [node.module]
            for nm in names:
                top = nm.split(".")[0]
                assert top != "oracle", f"{path} imports the oracle"
                # torch.distributed is rendezvous / barrier plumbing of the multi-GPU helpers only (parallel.py)
                banned = ("triton", "cupy", "numba") + (() if path.name == "parallel.py" else ("torch",))
                assert top not in banned, f"{path} imports {top}"
                if top == "scipy":
                    scipy_sites.append(path.name)
    # set-level scalar host work on RESULT rows, exactly the calls the reference makes there: optimize.minimize over the back-projection
    # segments (winston_lutz.py:1614-1640) and Rotation.as_euler for a non-default axes order of align_points (winston_lutz.py:3655-3658)
    assert sorted(scipy_sites) == ["winston_lutz.py", "winston_lutz_mtmf.py"], scipy_sites
