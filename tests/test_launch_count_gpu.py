"""Engine.launches (the benchmark's gpu_launches) counts what the device ran: under torch.profiler with CUDA activity, the
kernels of namespace mv2 each case ran equal the sum of the `launches` added by every engine the case used (the tokenizer's,
the discriminator's and the VGG's).  The library counts its own launches (mv2_launch_count) and Engine._call adds the
change over each call, so no literal per entry point can go stale.

Cases: the README tokenize + decode in bf16 (fused and unfused ResidualUnits, bf16 linear attention, slab / down-space
convs, the channels-first conv_out) and its layers in fp32 at 32 px (CUDA-core conv, fp32 linear attention, unfused
GEGLU, fp32 SqueezeExcite); a README training step with GAN, VGG and attention dropout (dropout kernels and mask, mse,
max-pool and its backward, the dense LFQ partials, the tap-wise discriminator convs, the data gradients); a 2^18-code LFQ
training forward + backward (the bit-factorised partials, finalize and backward); FSQ; streamed tokenize / decode of the
cond_wide, gateloop and sff configs of tests/test_option_calls_cpu.py and a whole-clip pad_reflect call; and CUDA-graph
capture and replay, which add what the eager call adds.  The last test asserts that the cases called every launching
entry point of the C ABI through Engine._call.

Each profiled case runs in a process of its own with one profiler session: after earlier sessions in a process (other
tests' or another case's), the first device records of a new session can be missing from its events."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import synth_data
from tests.test_option_calls_gpu import _inputs, _model, _run
from tests.test_stream_gpu import _decode_stream, _schedules, _tokenize_stream
from tests.test_train_calls_cpu import README_TRAIN_KW
from tests.util import ROOT, build_product, golden_video, load_golden

from magvit2_pytorch_b200 import VideoTokenizer, _lib
from magvit2_pytorch_b200.engine import Engine

pytestmark = pytest.mark.gpu

# entry points that launch nothing: queries return values, not status codes
NON_LAUNCHING = {"mv2_abi_version", "mv2_last_error", "mv2_device_arch", "mv2_launch_count", "mv2_set_pdl",
                 "mv2_tc_ru_records", "mv2_tc_slab_plan", "mv2_tc_slab_tile"}
LAUNCHING = {n for n in _lib.SIGNATURES
             if n not in NON_LAUNCHING and not re.search(r"_supported$|_workspace_bytes$", n)}

SEEN = set()       # entry points Engine._call was given, over all cases
RAN = set()        # cases that ran


def _profiled(engines, run):
    """Runs run() under torch.profiler -> (launches `engines` added, mv2 kernels the device ran)."""
    torch.cuda.synchronize()
    l0 = [e.launches for e in engines]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "mv2::" in e.name)
    return sum(e.launches - n for e, n in zip(engines, l0)), kernels


def _readme(dtype, **kw):
    g = load_golden("readme")
    m = build_product(dict(g["kwargs"], **kw), g["wseed"]).cuda().to(dtype)
    return m, golden_video(g)


def _eval_call(m, video):
    with torch.no_grad():
        m.decode_from_code_indices(m.tokenize(video))


def case_readme_bf16():
    m, video = _readme(torch.bfloat16)
    return _profiled([m.engine], lambda: _eval_call(m, video.cuda()))


def case_readme_layers_fp32():
    m, _ = _readme(torch.float32, image_size=32)
    video = synth_data.synth_video(1, 3, 17, 32).cuda()
    return _profiled([m.engine], lambda: _eval_call(m, video))


def case_train_step():
    torch.manual_seed(0)
    m = VideoTokenizer(**README_TRAIN_KW, attn_dropout=0.1, vgg=synth_data.build_vgg(synth_data.VGG16_CFG, 4096))
    synth_data.fill_state_dict_(m)
    synth_data.fill_discr_(m)
    synth_data.fill_vgg_(m.vgg)
    m = m.cuda().bfloat16().train()
    m.vgg.eval()
    video = synth_data.synth_video(2, 3, 17, 128).cuda().bfloat16()

    def step():
        loss, _ = m(video, return_loss=True)
        loss.backward()
        loss, _ = m(video, return_discr_loss=True, apply_gradient_penalty=False)
        loss.backward()

    torch.manual_seed(1)
    step()                      # warm-up: the discriminator's and the VGG's packs and engines
    torch.manual_seed(2)
    return _profiled([m.engine, m.discr._pack_cache.engine, m._vgg_cache.engine], step)


def case_lfq_2_18_train():
    g = load_golden("mini_lfq18_train")
    m = build_product(g["kwargs"], g["wseed"]).cuda().train()
    video = golden_video(g).cuda()

    def step():
        total, _ = m(video, return_loss=True)
        total.backward()
    return _profiled([m.engine], step)


def case_fsq():
    m = _model("fsq")
    video, cond, ff = _inputs("fsq", m)
    return _profiled([m.engine], lambda: _run(m, video, cond, ff))


def case_stream_and_pad_reflect():
    models = {name: _model(name) for name in ("cond_wide", "gateloop", "sff", "pad_reflect")}
    inputs = {name: _inputs(name, m) for name, m in models.items()}

    def run():
        for name, m in models.items():
            video, cond, ff = inputs[name]
            codes, _ = _run(m, video, cond, ff)
            if name == "pad_reflect":
                continue
            n_lat = codes.shape[1]
            with torch.no_grad():
                _tokenize_stream(m, video, _schedules(m.time_downsample_factor, n_lat, ff)[1], cond, ff)
                _decode_stream(m, codes, [1] * n_lat, cond, ff)
    return _profiled([m.engine for m in models.values()], run)


CASES = {f.__name__[5:]: f for f in (case_readme_bf16, case_readme_layers_fp32, case_train_step, case_lfq_2_18_train,
                                     case_fsq, case_stream_and_pad_reflect)}


def _child(name):
    """Runs case `name` in this process, recording the entry points Engine._call is given, and prints the result."""
    seen, call = set(), Engine._call

    def recording(self, entry, *args, stream=None):
        seen.add(entry)
        return call(self, entry, *args, stream=stream)
    Engine._call = recording
    launches, kernels = CASES[name]()
    print("RESULT " + json.dumps(dict(launches=launches, kernels=kernels, entries=sorted(seen))), flush=True)


def _run_case(name):
    """Case `name` in a child process -> (launches, kernels); records its entry points in SEEN."""
    torch.cuda.empty_cache()
    code = f"import sys; sys.path.insert(0, {ROOT!r}); import tests.test_launch_count_gpu as L; L._child({name!r})"
    p = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    res = [line for line in p.stdout.splitlines() if line.startswith("RESULT ")]
    assert p.returncode == 0 and res, (p.returncode, p.stdout[-4000:], p.stderr[-4000:])
    r = json.loads(res[-1][len("RESULT "):])
    SEEN.update(r["entries"])
    RAN.add(name)
    return r["launches"], r["kernels"]


@pytest.mark.parametrize("name", list(CASES))
def test_launches_equal_profiled_kernels(name):
    launches, kernels = _run_case(name)
    assert kernels > 0 and launches == kernels, (launches, kernels)
    print(f"\n{name}: {kernels} kernels launched and counted")


def test_cuda_graph_capture_and_replay_count_the_eager_launches():
    """With cuda_graphs on, the plain first call, the capture and each replay add to launches what the eager call adds."""
    m, video = _readme(torch.bfloat16)
    video = video.cuda()
    eng = m.engine
    with torch.no_grad():
        codes = m.tokenize(video)

    def added(fn):
        torch.cuda.synchronize()
        l0 = eng.launches
        with torch.no_grad():
            fn()
        torch.cuda.synchronize()
        return eng.launches - l0

    calls = (lambda: m.tokenize(video), lambda: m.decode_from_code_indices(codes))
    eager = [added(fn) for fn in calls]
    m.cuda_graphs = True
    for fn, n in zip(calls, eager):
        assert n > 0 and [added(fn) for _ in range(3)] == [n] * 3, n      # plain call, capture, replay
    assert m._graphs and all(v != "warm" for v in m._graphs.values())


def test_cases_call_every_launching_entry_point():
    """Every launching entry point of the C ABI was called through Engine._call by the cases above (run here when they
    did not run in this session)."""
    for name in CASES:
        if name not in RAN:
            _run_case(name)
    assert SEEN == LAUNCHING, (sorted(LAUNCHING - SEEN), sorted(SEEN - LAUNCHING))
