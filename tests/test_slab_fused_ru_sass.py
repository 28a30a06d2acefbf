"""The fused ResidualUnit launch (mv2_tc_ru_forward, slab kernel flavour EPI_FUSED_RU = 5) runs both epilogues on the
accumulator fragments and stores y with TMA.

Without a GPU, on the built library: the fused instances store y with bulk tensor stores, their only global stores are
the SqueezeExcite pool records (4- and 8-byte stores of fp32 values; y used to leave as 16-byte row pieces), and they
have no stack frame.

On the GPU: the fused launch's y equals the unfused slab path's conv1(ELU(conv3(x))) bit for bit: both run the same
MMAs in the same K order and the same per-element epilogue math.  The shapes are the benchmark's units (README config,
fewer frames) and planes whose H and W are not multiples of the macro tile (16 x 8 mw), where TMA clips the boxes."""
import ctypes as C
import re

import pytest
import torch

from magvit2_pytorch_b200._lib import ACT_ELU, TcRuArgs
from tests.test_slab_pipeline import _dump

FUSED = 5
NAME = re.compile(r"tc_slab_kernelILi(\d+)ELi(\d+)E")
STG = re.compile(r"(@!?U?P\w+\s+)?(STG\S*)")


@pytest.fixture(scope="module")
def sass():
    """{N tile: SASS instructions} of the fused instances"""
    out = {}
    for block in re.split(r"\n\s*Function : ", _dump("-sass"))[1:]:
        name, body = block.split("\n", 1)
        m = NAME.search(name)
        if m and int(m.group(1)) == FUSED:
            out[int(m.group(2))] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    assert sorted(out) == [32, 64, 128], sorted(out)
    return out


def test_y_through_tma(sass):
    for bn, ins in sass.items():
        assert any(re.search(r"\bUTMASTG\b", i) for i in ins), bn
        stores = {STG.match(i).group(2) for i in ins if STG.match(i)}
        assert stores <= {"STG.E", "STG.E.64"}, (bn, stores)


def test_no_stack_frame():
    usage = [(name, line) for name, line in re.findall(r"Function (\S*tc_slab_kernel\S*):\s*\n\s*(.*)", _dump("-res-usage"))
             if int(NAME.search(name).group(1)) == FUSED]
    assert len(usage) == 3
    for name, line in usage:
        assert "STACK:0 " in line, (name, line)


RU_Y_CASES = [
    # name, C, (B, T, H, W)
    ("readme_c64_128x128", 64, (1, 3, 128, 128)),
    ("readme_c128_64x64", 128, (2, 3, 64, 64)),
    ("c64_ragged_20x36", 64, (1, 3, 20, 36)),
    ("c64_ragged_9x9", 64, (2, 2, 9, 9)),
    ("c128_ragged_20x12", 128, (1, 4, 20, 12)),
    ("c128_ragged_33x17", 128, (1, 2, 33, 17)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", RU_Y_CASES, ids=[c[0] for c in RU_Y_CASES])
def test_fused_y_equals_unfused(case):
    from tests.test_tc_conv_gpu import _engine, _ru_pack

    assert torch.cuda.is_available()
    name, C_, (B, T, H, W) = case
    g = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    p, _ = _ru_pack(C_, g)
    x = torch.randn((B, T, H, W, C_), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    eng.use_tc, eng.tc_variant = True, "auto"
    c3, c1 = p["conv3"], p["conv1"]
    ra = TcRuArgs(x=x.data_ptr(), w3=c3.w_tc.data_ptr(), b3=c3.bias_tc.data_ptr(), w1=c1.w_tc.data_ptr(),
                  b1=c1.bias_tc.data_ptr(), se_wk=p["wk"].data_ptr(), se_bk=p["bk"], y=None, se_ws=None,
                  B=B, T=T, H=H, W=W, C=C_, kt=3, kh=3, kw=3)
    assert eng.lib.mv2_tc_ru_supported(C.byref(ra)), name
    y = torch.full_like(x, float("nan"))
    ws = torch.empty(eng.lib.mv2_tc_ru_workspace_bytes(C.byref(ra)) // 4, device="cuda", dtype=torch.float32)
    ra.y, ra.se_ws = y.data_ptr(), ws.data_ptr()
    eng._call("mv2_tc_ru_forward", C.byref(ra), None)
    eng.slab_calls = 0
    y_ref = eng.conv(eng.conv(x, c3, act=ACT_ELU), c1, act=ACT_ELU)
    torch.cuda.synchronize()
    assert eng.slab_calls == 2, "the unfused convs did not run on the slab kernel"
    assert torch.equal(y, y_ref), (name, (y.float() - y_ref.float()).abs().max().item(), (y != y_ref).float().mean().item())
