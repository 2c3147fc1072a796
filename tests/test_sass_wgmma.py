"""The tensor-core convolution kernels as compiled: every k_conv_halo / k_conv_tc instantiation of libdfvo_b200.so must keep one
tap's wgmma group in flight while the next one is issued.

The MMA loops commit one wgmma group per tap (per ring stage in k_conv_tc) and wait with wgmma.wait_group 1.  If a run-time branch
sits between a group's wgmma.fence and its commit, ptxas closes a group inside every branch, reports "C7519 warpgroup.arrive is
injected", and the commit becomes a second, empty group (`HGMMA.64x8x16 ... RZ, gdesc[URZ], RZ, !UPT, gsb0`).  The wait then
lets only that empty group stay in flight, and the tensor pipe drains after every tap.  This test reads the SASS and ptxas'
notes (csrc/build.log) so that an edit to the loops cannot quietly bring the drain back.  It needs the CUDA toolkit, not a GPU."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "df-vo_b200", "csrc")
KERNEL = re.compile(r"_ZN4dfvo(11k_conv_halo|9k_conv_tc)I")


def _toolkit():
    nvcc = shutil.which("nvcc")
    if nvcc is None:
        return None
    cuobjdump = os.path.join(os.path.dirname(os.path.realpath(nvcc)), "cuobjdump")
    return cuobjdump if os.path.exists(cuobjdump) else shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def built():
    cuobjdump = _toolkit()
    if cuobjdump is None:
        pytest.skip("the CUDA toolkit (nvcc, cuobjdump) is not installed")
    spec = importlib.util.spec_from_file_location("_dfvo_build", os.path.join(CSRC, "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    lib = m.build()
    log = os.path.join(CSRC, "build.log")
    if not os.path.exists(log):                      # the library is current but its ptxas log is gone: compile again
        lib = m.build(force=True)
    sass = subprocess.run([cuobjdump, "-sass", lib], check=True, capture_output=True, text=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", sass)
    funcs = {name: body for name, body in zip(parts[1::2], parts[2::2]) if KERNEL.match(name)}
    return funcs, open(log).read()


def test_conv_kernels_present(built):
    funcs, _ = built
    assert any(n.startswith("_ZN4dfvo11k_conv_halo") for n in funcs), "no k_conv_halo in the SASS"
    assert any(n.startswith("_ZN4dfvo9k_conv_tc") for n in funcs), "no k_conv_tc in the SASS"


def test_no_empty_wgmma_group(built):
    funcs, _ = built
    bad = {n: len(re.findall(r"HGMMA\.\S+ RZ, gdesc\[URZ\]", body)) for n, body in funcs.items()}
    assert not any(bad.values()), "empty HGMMA groups: %s" % {n: c for n, c in bad.items() if c}


def test_one_group_stays_in_flight(built):
    funcs, _ = built
    missing = [n for n, body in funcs.items() if "WARPGROUP.DEPBAR.LE gsb0, 0x1" not in body]
    assert not missing, "no WARPGROUP.DEPBAR.LE gsb0, 0x1 in %s" % missing


def test_ptxas_notes(built):
    funcs, log = built
    notes = [l for l in log.splitlines() if re.search(r"\(C75(19|10)\)", l) and KERNEL.search(l)]
    assert not notes, "ptxas wgmma notes:\n" + "\n".join(notes[:10])
    props = dict(re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores", log))
    for name in funcs:
        assert name in props, "%s is not in build.log" % name
    spills = {n: int(s) for n, s in props.items() if KERNEL.match(n) and int(s)}
    assert not spills, "spills: %s" % spills
