"""The C-ABI library loads and exports every symbol include/magvit2_b200.h declares (no compute)."""
import ctypes
import os
import re

import pytest

from magvit2_pytorch_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "magvit2_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mv2_[a-z0-9_]+)\s*\(", src)))


def test_library_built():
    assert os.path.isfile(_lib.LIB_PATH), "run __graft_entry__.build() first"


def test_every_declared_symbol_is_exported_and_bound():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature in _lib.py"
    for name in _lib.SIGNATURES:
        assert name in declared, f"{name} bound in _lib.py but not declared in the header"


def test_load_and_abi_version_5():
    """ABI version 5: the library, the header's MV2_ABI_VERSION and the ctypes binding agree (load() checks the binding)."""
    lib = _lib.load()
    assert lib.mv2_abi_version() == 5
    header = open(os.path.join(ROOT, "include", "magvit2_b200.h")).read()
    assert int(re.search(r"#define\s+MV2_ABI_VERSION\s+(\d+)", header).group(1)) == 5
    assert lib.mv2_se_workspace_bytes(2, 256, 64) == (2 * 8 * 66 + 2 * 80) * 4
    assert lib.mv2_linattn_workspace_bytes(3, 16, 1024) == 3 * 16 * 4 * 657 * 4 + 3 * 16 * 2 * 16 * 88 * 2


def test_launch_count_is_per_thread_and_skips_refused_calls():
    """mv2_launch_count is exported and bound, reads 0 on a freshly started thread, and a call refused by its argument
    check (mv2_rmsnorm with x = NULL touches no CUDA API) returns MV2_E_ARG without counting a launch."""
    import threading
    lib = _lib.load()
    assert _lib.SIGNATURES["mv2_launch_count"] == (ctypes.c_uint64, [])
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "mv2_launch_count")
    seen = {}

    def run():
        seen["fresh"] = lib.mv2_launch_count()
        buf = (ctypes.c_float * 8)()
        seen["rc"] = lib.mv2_rmsnorm(None, ctypes.addressof(buf), _lib.MV2_F32, ctypes.addressof(buf), 1, 1, 1, 8, 0, None)
        seen["after"] = lib.mv2_launch_count()

    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert seen == {"fresh": 0, "rc": -1, "after": 0}, seen       # MV2_E_ARG = -1


def test_struct_sizes_match_header_layout():
    # 5 pointers + 22 int32 (conv), 3 pointers + 8 int32 + 3 int64 (attention)
    assert ctypes.sizeof(_lib.ConvArgs) == 5 * 8 + 22 * 4 + 8            # + oscale pointer
    assert ctypes.sizeof(_lib.TcConvArgs) == 5 * 8 + 22 * 4 + 8 + 8      # + oscale pointer, out_layout (+ tail padding)
    assert ctypes.sizeof(_lib.AttnArgs) == 3 * 8 + 8 * 4 + 3 * 8


def test_sass_is_sm90a():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_tensor_core_kernels_issue_wgmma_fed_by_tma():
    """Every instance of the slab and tap-wise conv kernels multiplies on the Hopper tensor cores (wgmma = HGMMA in the
    SASS) with operands brought in by TMA tensor loads (UTMALDG).  Static check on the SASS."""
    import re
    import subprocess
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    kernels = re.split(r"\n\s*Function : ", sass)[1:]
    checked = 0
    for k in kernels:
        name = k.split("\n", 1)[0]
        if "tc_slab_kernel" not in name and "tc_conv_kernel" not in name:
            continue
        ins = [l for l in k.splitlines() if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
        assert any("HGMMA" in l and "F32.BF16" in l for l in ins), f"{name}: no bf16 wgmma (HGMMA) in the SASS"
        assert any("UTMALDG" in l for l in ins), f"{name}: no TMA tensor loads (UTMALDG)"
        checked += 1
    assert checked >= 6 * 3       # 8 slab + 3 tap-kernel epilogue flavours, each for N tiles of 32 / 64 / 128
