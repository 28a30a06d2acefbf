"""SURVEY 8f N2 (first slice): ``model.train(); loss, _ = model(video, return_loss=True); loss.backward()`` -- the generator step of
the reference trainer (T:356-363) -- against the loss values and parameter gradients the UNMODIFIED reference produced on the same
weights and clip (tests/golden/mini_train.pt, oracle/make_train_golden.py)."""
import pytest
import torch

from tests.test_oracle import grad_digest_close
from tests.util import build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu


def _require_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _train_step(model, video, cond=None):
    model.train()
    for p in model.parameters():
        p.grad = None
    total, bd = model(video, return_loss=True) if cond is None else model(video, cond=cond, return_loss=True)
    assert total.requires_grad and total.grad_fn is not None
    total.backward()
    return total, bd


@pytest.mark.parametrize("name", ["mini_train", "mini_mc_train", "mini_fsq_train", "mini_gateloop_train", "mini_cond_train", "mini_sff_train", "pad_reflect_train", "pad_circular_train"])
def test_fp32_losses_and_gradients_vs_reference_golden(name):
    """LFQ (README-layer mini config), two spherical codebooks, FSQ (straight-through round), gateloop_time layers, and
    cond_residual layers (ResidualUnitMod / Conv3DMod + the cond stems)."""
    _require_cuda()
    g = load_golden(name)
    gt = g["train"]
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    cond = g["cond"].cuda() if g.get("cond") is not None else None
    total, bd = _train_step(model, golden_video(g).cuda(), cond)
    assert abs(total.item() - gt["total_loss"].item()) < 1e-5
    assert abs(bd.recon_loss.item() - gt["recon_loss"].item()) < 1e-5
    assert abs(float(bd.lfq_aux_loss.detach()) - float(gt["aux"])) < 1e-5
    if "per_sample_entropy" in gt:
        ps, be, cm = bd.quantizer_loss_breakdown
        for got, k in ((ps, "per_sample_entropy"), (be, "batch_entropy"), (cm, "commitment")):
            assert abs(got.item() - gt[k].item()) < 1e-5, k
    else:
        assert bd.quantizer_loss_breakdown is None
    named = dict(model.named_parameters())
    gnorm = sum(d["norm"] ** 2 for d in gt["grads"].values() if d is not None) ** 0.5
    worst, checked = 0.0, 0
    for k, dg in gt["grads"].items():
        if k not in named:
            continue
        p = named[k]
        if dg is None:      # parameters the reference's forward never touches
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        assert p.grad is not None, k
        worst = max(worst, grad_digest_close(p.grad, dg, 5e-3, k, atol=1e-7 * gnorm))
        checked += 1
    assert checked >= {"mini_train": 250, "mini_fsq_train": 250}.get(name, 50), checked
    print(f"{name}: {checked} parameter gradients checked, worst relative deviation vs the reference {worst:.2e}")


def test_own_dgrad_kernels_agree_with_the_library_dgrad():
    """The data gradient of the stride-1 causal convs runs on the engine's own conv kernels (flipped / transposed weights); with
    TrainRunner.own_dgrad switched off the same gradients come from aten.convolution_backward: both agree to fp32 round-off."""
    _require_cuda()
    from magvit2_pytorch_b200 import train as T
    g = load_golden("mini_train")
    video = golden_video(g).cuda()
    grads = []
    # the library side in true fp32: TF32 convolutions (cuDNN's default on this GPU) would round far above fp32 round-off
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for own in (True, False):
            model = build_product(g["kwargs"], g["wseed"]).cuda()
            orig = T.TrainRunner.__init__

            def patched(self, m, _own=own, _orig=orig):
                _orig(self, m)
                self.own_dgrad = _own
            T.TrainRunner.__init__ = patched
            try:
                _train_step(model, video)
            finally:
                T.TrainRunner.__init__ = orig
            grads.append({k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    worst = 0.0
    gnorm = sum(float(b.double().pow(2).sum()) for b in grads[1].values()) ** 0.5
    for k, a in grads[0].items():
        b = grads[1][k]
        # gradients that are mathematically zero (bias of a softmax logit) hold only round-off noise: absolute floor
        worst = max(worst, float((a - b).abs().max()) / (float(b.abs().max()) + 1e-6 * gnorm))
    print(f"own dgrad vs cuDNN dgrad: worst relative deviation {worst:.2e}")
    assert worst < 2e-3, worst


def test_optimizer_step_changes_the_loss_and_repacks_the_weights():
    """Trainer-shaped loop: backward, optimizer step, forward again -- the engine re-packs the updated parameters and the
    reconstruction loss goes down along the negative gradient by about lr * |grad|^2 (first-order prediction).  The quantiser's
    auxiliary loss is switched off here: its inv_temperature = 100 softmax makes the loss surface too sharp for a fixed step."""
    _require_cuda()
    g = load_golden("mini_train")
    model = build_product(dict(g["kwargs"], quantizer_aux_loss_weight=0.), g["wseed"]).cuda()
    video = golden_video(g).cuda()
    lr = 2e-6
    opt = torch.optim.SGD(model.parameters(), lr=lr)
    losses, gsq = [], []
    for _ in range(3):
        total, _ = _train_step(model, video)
        gsq.append(sum(float(p.grad.double().pow(2).sum()) for p in model.parameters() if p.grad is not None))
        opt.step()
        losses.append(total.item())
    print("losses", losses, "predicted first step", -lr * gsq[0])
    assert losses[1] < losses[0] and losses[2] < losses[1], losses
    pred = -lr * gsq[0]
    # the straight-through estimator is not the true gradient of the encoder side, so the decrease is smaller than predicted
    assert 0.05 * pred > losses[1] - losses[0] > 3.0 * pred, (losses, pred)
    model.eval()
    with torch.no_grad():
        codes = model.tokenize(video)            # the inference path still runs on the updated weights
    assert codes.dtype == torch.int64


def test_bf16_gradients_agree_with_fp32():
    """bf16 training path (wgmma forward, cuDNN bf16 backward) against the fp32 path on the reconstruction loss.  (With the LFQ
    auxiliary loss the comparison is meaningless: its logits are 200 x the pre-sign values, so bf16 round-off of the encoder
    output changes the code probabilities by O(1) -- in the reference's own bf16 run as well.)"""
    _require_cuda()
    g = load_golden("mini_train")
    video = golden_video(g).cuda()
    kw = dict(g["kwargs"], quantizer_aux_loss_weight=0.)
    m32 = build_product(kw, g["wseed"]).cuda()
    m16 = build_product(kw, g["wseed"]).cuda().bfloat16()
    t32, _ = _train_step(m32, video)
    t16, _ = _train_step(m16, video.bfloat16())
    assert abs(t16.float().item() - t32.item()) < 0.05 * abs(t32.item()) + 0.05

    def cosine(prefixes):
        num = den_a = den_b = 0.0
        for (k, a), (_, b) in zip(m32.named_parameters(), m16.named_parameters()):
            if a.grad is None or b.grad is None or not k.startswith(prefixes):
                continue
            ga, gb = a.grad.double().flatten(), b.grad.double().flatten()
            num += float(ga @ gb); den_a += float(ga @ ga); den_b += float(gb @ gb)
        return num / (den_a ** 0.5 * den_b ** 0.5)

    cos_dec = cosine(("decoder_layers", "conv_out", "quantizers.project_out"))
    cos_enc = cosine(("encoder_layers", "conv_in", "quantizers.project_in"))
    print(f"cosine(fp32 grads, bf16 grads): decoder side {cos_dec:.4f}, encoder side {cos_enc:.4f}")
    assert cos_dec > 0.95, cos_dec
    assert cos_enc > 0.5, cos_enc


def test_generator_step_under_distributed_data_parallel():
    """The trainer wraps the tokenizer in DistributedDataParallel (accelerate, find_unused_parameters=True as the reference's dead
    final LayerNorm requires): the custom autograd Function spanning the model must feed DDP's reducer a gradient for every
    parameter it reaches.  World size 1 (NCCL): gradients equal the plain run's, and a second step works (reducer finalised)."""
    _require_cuda()
    import socket
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    if dist.is_initialized():
        pytest.skip("a process group is already initialised in this process")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    g = load_golden("mini_train")
    video = golden_video(g).cuda()
    plain = build_product(g["kwargs"], g["wseed"]).cuda()
    _train_step(plain, video)
    want = {k: p.grad.clone() for k, p in plain.named_parameters() if p.grad is not None}
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        model = build_product(g["kwargs"], g["wseed"]).cuda()
        ddp = DDP(model, device_ids=[torch.cuda.current_device()], find_unused_parameters=True)
        ddp.train()
        for step in range(2):
            for p in model.parameters():
                p.grad = None
            loss, bd = ddp(video, return_loss=True)
            loss.backward()
        got = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
        assert set(want) <= set(got)
        for k, w in want.items():
            assert torch.allclose(got[k], w, rtol=1e-4, atol=1e-6 * float(w.abs().max()) + 1e-12), k
    finally:
        dist.destroy_process_group()
