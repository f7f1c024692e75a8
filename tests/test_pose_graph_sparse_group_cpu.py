"""CPU: the declarations of the grouped block-sparse LM step (sta_pg_group_plan_*, sta_pose_graph_lm_step_sparse_group),
the StaPgSparseStep layout of _lib.py against the C one, and the refusals that come before any device call."""
import ctypes
import os
import re
import subprocess

import pytest

from conftest import ROOT
from vista_slam_b200 import _lib

HEADER = os.path.join(ROOT, "include", "sta_b200.h")
NEW = ("sta_pg_group_plan_create", "sta_pg_group_plan_destroy", "sta_pg_group_plan_info",
       "sta_pose_graph_lm_step_sparse_group")


def test_header_declares_and_library_exports_the_group_entry_points():
    hdr = open(HEADER).read()
    L = _lib.lib()
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(L, name), name
    assert "typedef struct StaPgSparseStep" in hdr and "STA_PG_GROUP_MAX = 16" in hdr
    assert _lib.PG_GROUP_MAX == 16


def test_sparse_step_layout_matches_c(tmp_path):
    """Field offsets and size of StaPgSparseStep, as a host C compiler lays the header's struct out."""
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "sta_b200.h"\nint main(void) {\n'
                   + "".join('  printf("%%s %%zu\\n", "%s", offsetof(StaPgSparseStep, %s));\n' % (f, f)
                             for f, _ in _lib.StaPgSparseStep._fields_)
                   + '  printf("size %zu\\n", sizeof(StaPgSparseStep));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    cc = next((c for c in ("cc", "gcc", "clang") if subprocess.run(["which", c], capture_output=True).returncode == 0), None)
    if cc is None:
        pytest.skip("no host C compiler")
    subprocess.run([cc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True)
               .stdout.splitlines())
    for f, _ in _lib.StaPgSparseStep._fields_:
        assert int(got[f]) == getattr(_lib.StaPgSparseStep, f).offset, f
    assert int(got["size"]) == ctypes.sizeof(_lib.StaPgSparseStep) == 48


FAKE = 4096  # stands for a plan or device pointer; never dereferenced by the refusals below


@pytest.mark.parametrize("case", ["null_out", "null_table", "G0", "G17", "G_negative", "null_member"])
def test_group_plan_create_refusals(case):
    L = _lib.lib()
    G = 2
    tab = (ctypes.c_void_p * 17)(*[FAKE + 256 * k for k in range(17)])
    out = ctypes.c_void_p(FAKE)
    out_p = ctypes.byref(out)
    msg = b"requirement failed"
    if case == "null_out":
        out_p = None
    elif case == "null_table":
        tab, msg = None, b"null plan table"
    elif case == "G0":
        G, msg = 0, b"STA_PG_GROUP_MAX"
    elif case == "G17":
        G, msg = 17, b"STA_PG_GROUP_MAX"
    elif case == "G_negative":
        G, msg = -1, b"STA_PG_GROUP_MAX"
    else:
        tab[1], msg = None, b"null plan"
    assert L.sta_pg_group_plan_create(tab, G, out_p) == 2
    assert msg in L.sta_last_error()
    if case != "null_out":
        assert out.value is None  # *out cleared before any check on the table


def test_group_plan_create_refuses_a_plan_named_twice():
    L = _lib.lib()
    tab = (ctypes.c_void_p * 3)(FAKE, FAKE + 256, FAKE)
    out = ctypes.c_void_p()
    assert L.sta_pg_group_plan_create(tab, 3, ctypes.byref(out)) == 2
    assert b"named twice" in L.sta_last_error() and out.value is None


def test_group_step_and_info_refuse_null_pointers():
    L = _lib.lib()
    steps = (_lib.StaPgSparseStep * 1)()
    info = ctypes.c_void_p(FAKE)
    assert L.sta_pose_graph_lm_step_sparse_group(None, steps, 1e-6, 1e32, info, None) == 2
    assert b"null pointer" in L.sta_last_error()
    assert L.sta_pg_group_plan_info(None, (ctypes.c_int64 * 4)()) == 2
    assert b"null argument" in L.sta_last_error()
    L.sta_pg_group_plan_destroy(None)  # a no-op
