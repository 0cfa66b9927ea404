"""Compile-time guard on the register sliding-window scatter (`window_consume2`, csrc/fmpm_scatter.cuh).

Every kernel that runs the scatter's node loop is compiled for sm_90a with `-Xptxas -v`, and its spill bytes are held to a budget:
the forward kernel `k_fwd<*, false, *>` must not spill at all (local-memory traffic inside the node loop costs the hot kernel more than
the loop's own arithmetic), and no other user of the loop may spill more than the figures below (CUDA 12.9).  Needs nvcc, no GPU."""
import importlib.util
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fluidlab_b200", "csrc")
# the library's own build settings (flags, FMPM_DEFS, nvcc), loaded from the file so that the package itself is not imported
_spec = importlib.util.spec_from_file_location("_fmpm_build", os.path.join(CSRC, "build.py"))
BUILD = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(BUILD)


def _nvcc():
    return BUILD.NVCC if os.path.exists(BUILD.NVCC) else shutil.which("nvcc")


# (spill stores, spill loads) in bytes per instantiation, keyed by the demangled template name; the spills that remain lie outside the
# node loop.  The other instantiations of `k_fwd<*, true, *>` (the lazy in-kernel grid_op) are not built.
BUDGET = {
    "k_fwd<0, false, false>": (0, 0),
    "k_fwd<0, false, true>": (0, 0),
    "k_fwd<1, false, false>": (0, 0),
    "k_fwd<1, false, true>": (0, 0),
    "k_fwd<0, true, false>": (24, 28),
    "k_fwd<1, true, false>": (0, 0),
    "k_p2g<false, false>": (0, 0),
    "k_p2g<false, true>": (0, 0),
    "k_p2g<true, false>": (0, 0),
    "k_p2g<true, true>": (0, 0),
    "k_g2p2g<false, false>": (0, 0),
    "k_g2p2g<false, true>": (4, 8),
    "k_g2p2g<true, false>": (0, 0),
    "k_g2p2g<true, true>": (4, 12),
    "k_g2p_grad_scatter<false>": (0, 0),
    "k_g2p_grad_scatter<true>": (0, 0),
}
_MANGLED = re.compile(r"_Z\d+(k_fwd|k_p2g|k_g2p2g|k_g2p_grad_scatter)I((?:L[ib]\d+E)+)E")


def _demangle(sym):
    m = _MANGLED.match(sym)
    if m is None:
        return None
    args = re.findall(r"L([ib])(\d+)E", m.group(2))
    return "%s<%s>" % (m.group(1), ", ".join(v if t == "i" else ("true" if v == "1" else "false") for t, v in args))


def _spills(src, out_dir):
    """{demangled kernel: (spill stores, spill loads)} from `ptxas -v` for one translation unit"""
    cmd = [_nvcc()] + BUILD.FLAGS + ["-Xptxas", "-v", "-cubin", os.path.join(CSRC, src), "-o", os.path.join(out_dir, src + ".cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    res, name = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = _demangle(m.group(1))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name is not None:
            res[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    return res


@pytest.fixture(scope="module")
def spills(tmp_path_factory):
    if _nvcc() is None:
        pytest.skip("nvcc not found")
    out = str(tmp_path_factory.mktemp("sass_budget"))
    with ThreadPoolExecutor(2) as ex:
        parts = list(ex.map(lambda s: _spills(s, out), ["fmpm_forward.cu", "fmpm_backward.cu"]))
    return {**parts[0], **parts[1]}


def test_every_scatter_kernel_is_compiled(spills):
    assert set(BUDGET) <= set(spills), sorted(set(BUDGET) - set(spills))


@pytest.mark.parametrize("kernel", sorted(BUDGET))
def test_scatter_kernel_spills_within_budget(spills, kernel):
    st, ld = spills[kernel]
    bst, bld = BUDGET[kernel]
    assert st <= bst and ld <= bld, f"{kernel}: {st} B spill stores / {ld} B spill loads, budget {bst} / {bld}"
