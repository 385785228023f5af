"""Build-artifact checks that need no GPU: the shipped libb200sparse.so carries sm_90a SASS with the
instruction forms DESIGN.md claims for the SpMV hot path (SURVEY §8 row a3) — TMA bulk copies and mbarrier
traffic in the pipe kernel, L1-bypassing 16-byte cp.async gathers in the async-gather kernel — and none of
the LDGSTS mis-encoding ptxas 12.9 produced for one variant of that kernel (see csrc/Makefile)."""
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(__file__)), "legate-sparse_b200", "lib", "libb200sparse.so")


@pytest.fixture(scope="module")
def sass():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[:500]
    return out.stdout


def functions(sass_text):
    """{mangled function name: its SASS text}"""
    parts = re.split(r"^\s*Function : ", sass_text, flags=re.M)
    return {p.split("\n", 1)[0].strip(): p for p in parts[1:]}


def test_sass_is_sm90a_and_has_the_claimed_instruction_forms(sass):
    assert "sm_90a" in sass
    fn = functions(sass)
    pipe = [t for n, t in fn.items() if "spmv_pipe_kernel" in n]
    ag = [t for n, t in fn.items() if "spmv_agather_kernel" in n]
    assert pipe and ag
    # pipe kernel: TMA bulk copies paced by mbarriers, cross-proxy fence before a stage is refilled
    assert all("UBLKCP.S.G" in t and "SYNCS.ARRIVE.TRANS64" in t and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in t for t in pipe)
    assert any("FENCE.VIEW.ASYNC" in t for t in pipe)
    # async-gather kernel: every instance gathers with the L1-bypassing 16-byte cp.async, streams with
    # no-allocate 128-bit loads, fetches its row pointers by TMA, and has no local-memory traffic (no spills)
    for t in ag:
        assert "LDGSTS.E.BYPASS.128" in t
        assert "LDG.E.NA.128" in t
        assert "UBLKCP.S.G" in t
        assert "LDGDEPBAR" in t and "DEPBAR.LE" in t
        assert " LDL" not in t and " STL" not in t
    # no tensor-core expectation on this path, and no leftovers of other architectures
    assert "wgmma" not in sass.lower()


def test_no_ldgsts_with_an_odd_descriptor_register(sass):
    """ptxas 12.9 encoded the gathers of an experimental variant as LDGSTS [R+UR0], desc[UR1] with UR0/UR1 never
    written (illegal instruction at run time).  An L2-hint descriptor is an even uniform-register pair."""
    bad = [l for l in sass.splitlines() if "LDGSTS" in l and re.search(r"desc\[UR\d*[13579]\]", l)]
    assert not bad, bad[:3]
