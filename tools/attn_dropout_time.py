"""Times attention dropout against plain attention at the tokenizer's attention shapes: mv2_attention and
mv2_attention_dropout (p = 0.1) in bf16 and fp32, and mv2_attention_dropout_mask (what the training backward regenerates),
at the space and time attention calls of the README config (4 clips x 17 frames x 128^2) and of cfg4 (1 clip x 17 frames
x 256^2); 8 heads of 32, 4 memory key/values.

Device events after a warm-up; prints the card's name and power limit with the numbers.

    python tools/attn_dropout_time.py [--iters 50]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from magvit2_pytorch_b200 import _lib  # noqa: E402

HEADS, DH, N_MEM = 8, 32, 4
# name, clips, frames at the layer, H W at the layer, axis
SHAPES = [("readme space", 4, 20, 256, "space"), ("readme time", 4, 5, 256, "time"),
          ("cfg4 space", 1, 20, 1024, "space"), ("cfg4 time", 1, 5, 1024, "time")]


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    print(f"card: {_card()}")
    print(f"{'shape':<14}{'dtype':<6}{'attention us':>14}{'dropout us':>12}{'ratio':>8}{'mask us':>10}")
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, B, T, HW, axis in SHAPES:
        n_tok = B * T * HW
        if axis == "space":
            lay = dict(n_outer=B * T, n_inner=1, L=HW, outer_stride=HW, inner_stride=0, tok_stride=1)
        else:
            lay = dict(n_outer=B, n_inner=HW, L=T, outer_stride=T * HW, inner_stride=1, tok_stride=HW)
        n_seq, L = lay["n_outer"] * lay["n_inner"], lay["L"]
        mem = torch.randn((2, HEADS, N_MEM, DH), generator=g, device="cuda")
        keep = torch.empty((n_seq, HEADS, L, N_MEM + L), dtype=torch.uint8, device="cuda")
        drop = _lib.DropoutArgs(seed=1234, call=0, p=0.1)
        t_mask = _time(lambda: _lib.check(lib.mv2_attention_dropout_mask(n_seq, HEADS, L, N_MEM, C.byref(drop), keep.data_ptr(), st)),
                       args.iters)
        for dt, code in ((torch.bfloat16, _lib.MV2_BF16), (torch.float32, _lib.MV2_F32)):
            qkv = torch.randn((n_tok, 3 * HEADS * DH), generator=g, device="cuda").to(dt)
            out = torch.empty((n_tok, HEADS * DH), device="cuda", dtype=dt)
            a = _lib.AttnArgs(qkv=qkv.data_ptr(), out=out.data_ptr(), mem_kv=mem.data_ptr(), dtype=code, heads=HEADS, dim_head=DH,
                              n_mem=N_MEM, causal=int(axis == "time"), **lay)
            t_plain = _time(lambda: _lib.check(lib.mv2_attention(C.byref(a), st)), args.iters)
            t_drop = _time(lambda: _lib.check(lib.mv2_attention_dropout(C.byref(a), C.byref(drop), st)), args.iters)
            print(f"{name:<14}{'bf16' if code else 'fp32':<6}{t_plain:>14.1f}{t_drop:>12.1f}{t_drop / t_plain:>8.2f}{t_mask:>10.1f}")


if __name__ == "__main__":
    main()
