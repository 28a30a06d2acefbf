"""Code-generation checks of the slab conv kernel's TMA-store epilogue on the built library, with cuobjdump and without a
GPU: the instances of the plain, GEGLU, residual and SpatialDownsample2x flavours (EPI_PLAIN = 0, EPI_GEGLU = 1,
EPI_PLAIN_RES = 4, EPI_DOWN_SPACE = 7) write their output with bulk tensor stores and no global store instruction, the
residual flavour loads its residual with TMA as well, and none of them has a stack frame."""
import re

import pytest

from tests.test_slab_pipeline import _dump

TMA_STORE_MODES = (0, 1, 4, 7)
NAME = re.compile(r"tc_slab_kernelILi(\d+)ELi(\d+)E")


@pytest.fixture(scope="module")
def sass():
    """{(epilogue flavour, N tile): SASS instructions} of the TMA-store instances"""
    out = {}
    for block in re.split(r"\n\s*Function : ", _dump("-sass"))[1:]:
        name, body = block.split("\n", 1)
        m = NAME.search(name)
        if m and int(m.group(1)) in TMA_STORE_MODES:
            out[(int(m.group(1)), int(m.group(2)))] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    assert sorted(out) == [(m, bn) for m in TMA_STORE_MODES for bn in (32, 64, 128)], sorted(out)
    return out


def test_bulk_tensor_stores_only(sass):
    for key, ins in sass.items():
        assert any(re.search(r"\bUTMASTG\b", i) for i in ins), key
        assert not [i for i in ins if re.match(r"(@!?U?P\w+\s+)?STG\b", i)], key


def test_residual_comes_through_tma(sass):
    loads = {key: sum(bool(re.search(r"\bUTMALDG\b", i)) for i in ins) for key, ins in sass.items()}
    for bn in (32, 64, 128):
        assert loads[(4, bn)] > loads[(0, bn)], loads


def test_no_stack_frame():
    usage = re.findall(r"Function (\S*tc_slab_kernel\S*):\s*\n\s*(.*)", _dump("-res-usage"))
    moved = [(name, line) for name, line in usage if int(NAME.search(name).group(1)) in TMA_STORE_MODES]
    assert len(moved) == 3 * len(TMA_STORE_MODES)
    for name, line in moved:
        assert "STACK:0 " in line, (name, line)
