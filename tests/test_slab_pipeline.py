"""Code-generation checks of the slab conv kernel on the built library, with cuobjdump and without a GPU: every
tc_slab_kernel instance keeps its accumulators in registers (no stack frame), splits the register file between the
producer and consumer warpgroups (setmaxnreg), and keeps one wgmma commit group in flight across ring stages."""
import os
import re
import shutil
import subprocess

import pytest

from magvit2_pytorch_b200 import _lib

N_INSTANCES = 8 * 3          # epilogue flavours x N tiles (32 / 64 / 128)


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        home = os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH") or "/usr/local/cuda"
        exe = os.path.join(home, "bin", "cuobjdump")
    if not os.path.isfile(exe):
        pytest.skip("cuobjdump not found")
    return exe


def _dump(*flags):
    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("library not built")
    return subprocess.run([_cuobjdump(), *flags, _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout


@pytest.fixture(scope="module")
def sass():
    """{mangled tc_slab_kernel name: its SASS}"""
    out = {}
    for block in re.split(r"\n\s*Function : ", _dump("-sass"))[1:]:
        name, body = block.split("\n", 1)
        if "tc_slab_kernel" in name:
            out[name.strip()] = body
    assert len(out) == N_INSTANCES, sorted(out)
    return out


def test_no_stack_frame():
    usage = re.findall(r"Function (\S*tc_slab_kernel\S*):\s*\n\s*(.*)", _dump("-res-usage"))
    assert len(usage) == N_INSTANCES
    for name, line in usage:
        assert "STACK:0 " in line, (name, line)


def test_register_split(sass):
    for name, body in sass.items():
        assert "USETMAXREG" in body, name


DUMMY_HGMMA = re.compile(r"HGMMA\.\S+ RZ, gdesc\[URZ\]")   # empty MMA ptxas adds to close a group it had to split


def _instructions(body):
    return [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]


def test_one_group_in_flight(sass):
    """Every depth-1 wait follows a whole commit group: WARPGROUP.ARRIVE, then real MMAs of which only the last carries
    gsb0.  A runtime branch inside a group makes ptxas split it (gsb0 on earlier MMAs) and close it with an empty MMA,
    so that the wait would leave nothing real in flight."""
    for name, body in sass.items():
        ins = _instructions(body)
        assert not any(DUMMY_HGMMA.search(i) for i in ins), name
        waits = [k for k, i in enumerate(ins) if re.match(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", i)]
        assert waits, name
        for k in waits:
            mmas = []
            for i in reversed(ins[:k]):
                if i.startswith("WARPGROUP."):
                    break
                if "HGMMA" in i:
                    mmas.append(i)
            assert mmas and "gsb0" in mmas[0], (name, k, mmas)
            assert not any("gsb0" in m for m in mmas[1:]), (name, k, mmas)
