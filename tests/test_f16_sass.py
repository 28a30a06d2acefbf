"""Code-generation checks of the fp16 instances of the tensor-core conv kernels on the built library, without a GPU: every
fp16 slab and tap-wise instance (tc_slab_f16_kernel, tc_conv_f16_kernel) multiplies with the fp16 form of wgmma
(HGMMA.64xNx16.F32 with no operand-type suffix; the bf16 form is HGMMA ... F32.BF16) fed by TMA tensor loads, never with the bf16 form, and has no stack frame; the fp16 forms of the
mma.sync attention kernels use the fp16 HMMA."""
import re

import pytest

from tests.test_slab_pipeline import _dump

NAME = re.compile(r"(tc_slab_f16_kernel|tc_conv_f16_kernel)ILi(\d+)ELi(\d+)E")


@pytest.fixture(scope="module")
def sass():
    out = {}
    for block in re.split(r"\n\s*Function : ", _dump("-sass"))[1:]:
        name, body = block.split("\n", 1)
        out[name.strip()] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    return out


def test_every_f16_conv_instance_uses_f16_wgmma(sass):
    found = {}
    for name, ins in sass.items():
        m = NAME.search(name)
        if not m:
            continue
        found[(m.group(1), int(m.group(2)), int(m.group(3)))] = ins
        assert any(re.match(r"HGMMA\.64x\d+x16\.F32 ", i) for i in ins), f"{name}: no fp16 wgmma"
        assert not any("HGMMA" in i and "BF16" in i for i in ins), f"{name}: bf16 wgmma in an fp16 instance"
        assert any("UTMALDG" in i for i in ins), f"{name}: no TMA tensor loads"
    slab = {(mode, bn) for k, mode, bn in found if k == "tc_slab_f16_kernel"}
    tap = {(mode, bn) for k, mode, bn in found if k == "tc_conv_f16_kernel"}
    # the same flavours and N tiles as the bf16 kernels: 8 slab flavours x 3 N tiles, 3 tap-wise flavours x 3
    assert len(slab) == 8 * 3 and len(tap) == 3 * 3, (sorted(slab), sorted(tap))


def test_f16_conv_instances_have_no_stack_frame():
    usage = re.findall(r"Function (\S*(?:tc_slab_f16_kernel|tc_conv_f16_kernel)\S*):\s*\n\s*(.*)", _dump("-res-usage"))
    assert len(usage) == 8 * 3 + 3 * 3
    for name, line in usage:
        assert "STACK:0 " in line, (name, line)


def test_f16_attention_mma_uses_f16_hmma(sass):
    names = [n for n in sass if "attention_mma_f16_kernel" in n or "attention_mma_dropout_f16_kernel" in n]
    assert len(names) == 4, names
    for n in names:
        assert any(re.match(r"HMMA\.16816\.F32(\s|$)", i) for i in sass[n]), n
        assert not any("HMMA.16816.F32.BF16" in i for i in sass[n]), n
