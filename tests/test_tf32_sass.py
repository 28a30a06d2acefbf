"""Code-generation checks of the TF32 instances of the tensor-core conv kernels on the built library, without a GPU: every
TF32 slab and tap-wise instance (tc_slab_tf32_kernel, tc_conv_tf32_kernel) multiplies with the TF32 form of wgmma
(HGMMA.64xNx8.F32.TF32) fed by TMA tensor loads, never with a 16-bit form, and has no stack frame.  The TF32 slab kernel has
the bf16 flavours and N tiles except the fused ResidualUnit (EPI_FUSED_RU = 5) and the transposed shuffle stores
(EPI_SHUFFLE_ST = 6), which DESIGN.md excludes."""
import re

import pytest

from tests.test_slab_pipeline import _dump

NAME = re.compile(r"(tc_slab_tf32_kernel|tc_conv_tf32_kernel|tc_slab_kernel|tc_conv_kernel)ILi(\d+)ELi(\d+)E")
EXCLUDED_SLAB_FLAVOURS = {5, 6}


@pytest.fixture(scope="module")
def sass():
    out = {}
    for block in re.split(r"\n\s*Function : ", _dump("-sass"))[1:]:
        name, body = block.split("\n", 1)
        out[name.strip()] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    return out


def _instances(sass, kernel):
    return {(int(m.group(2)), int(m.group(3))) for m in map(NAME.search, sass) if m and m.group(1) == kernel}


def test_every_tf32_conv_instance_uses_tf32_wgmma(sass):
    n = 0
    for name, ins in sass.items():
        m = NAME.search(name)
        if not m or "tf32" not in m.group(1):
            continue
        n += 1
        assert any(re.match(r"HGMMA\.64x\d+x8\.F32\.TF32 ", i) for i in ins), f"{name}: no TF32 wgmma"
        # ptxas closes a commit group at a branch with an empty MMA (zero descriptor and registers, "gdesc[URZ]"): no math
        assert not any(re.match(r"HGMMA\.64x\d+x16\.", i) and "gdesc[URZ]" not in i for i in ins), \
            f"{name}: 16-bit wgmma in a TF32 instance"
        assert any("UTMALDG" in i for i in ins), f"{name}: no TMA tensor loads"
    assert n > 0


def test_tf32_flavours_are_the_bf16_ones_less_the_exclusions(sass):
    bf16_slab, tf32_slab = _instances(sass, "tc_slab_kernel"), _instances(sass, "tc_slab_tf32_kernel")
    assert tf32_slab == {(mode, bn) for mode, bn in bf16_slab if mode not in EXCLUDED_SLAB_FLAVOURS}
    assert _instances(sass, "tc_conv_tf32_kernel") == _instances(sass, "tc_conv_kernel")
    assert len(tf32_slab) == 6 * 3


def test_tf32_conv_instances_have_no_stack_frame():
    usage = re.findall(r"Function (\S*(?:tc_slab_tf32_kernel|tc_conv_tf32_kernel)\S*):\s*\n\s*(.*)", _dump("-res-usage"))
    assert len(usage) == 6 * 3 + 3 * 3
    for name, line in usage:
        assert "STACK:0 " in line, (name, line)
