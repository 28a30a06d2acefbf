"""Host-side mirror of the reference's VideoTokenizer interface (no GPU needed)."""
import copy
import pickle

import pytest
import torch

from magvit2_pytorch_b200 import VideoTokenizer
from tests.util import README_LAYERS, build_product, load_golden


def test_schedule_readme():
    m = VideoTokenizer(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    assert m.time_downsample_factor == 4 and m.time_padding == 3 and m.fmap_size == 16
    dims = [(s.kind, s.dim, s.dim_out) for s in m.stages]
    assert dims[1] == ("compress_space", 64, 128) and dims[9] == ("compress_time", 512, 512)
    assert len(m.encoder_layers) == len(README_LAYERS) + 1       # + the dead LayerNorm (M:1322)
    assert len(m.decoder_layers) == len(README_LAYERS)
    n_params = sum(p.numel() for p in m.parameters())
    assert abs(n_params - 117.8e6) < 0.2e6                       # SURVEY.md 8: 117.8 M generator params
    assert isinstance(m.parameters(), list)


def test_state_dict_keys_follow_reference_layout():
    m = VideoTokenizer(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS)
    keys = set(m.state_dict().keys())
    for k in ["conv_in.conv.weight", "encoder_layers.0.fn.0.conv.bias", "encoder_layers.0.fn.4.to_k.weight",
              "encoder_layers.2.1.fn.4.net.2.weight", "encoder_layers.1.conv.weight", "decoder_layers.2.net.0.weight",
              "encoder_layers.8.0.fn.mem_kv", "encoder_layers.8.0.fn.to_qkv.0.weight", "encoder_layers.8.0.fn.to_out.1.weight",
              "encoder_layers.13.0.fn.fn.norm.gamma", "encoder_layers.13.1.fn.fn.net.2.bias",
              "encoder_layers.5.0.fn.attn.to_kv.0.weight", "encoder_layers.5.1.fn.norm.gamma",
              "encoder_layers.14.1.weight", "quantizers.mask", "quantizers.project_in.weight", "conv_out.conv.bias"]:
        assert k in keys, k
    assert "zero" not in keys
    assert m.state_dict()["quantizers.mask"].tolist() == [512, 256, 128, 64, 32, 16, 8, 4, 2, 1]


def test_constructor_errors():
    with pytest.raises(ValueError):
        VideoTokenizer(image_size=32, codebook_size=1024, layers=("bogus",))
    with pytest.raises(AssertionError):
        VideoTokenizer(image_size=32, layers=("residual",))                       # no codebook_size (M:1359)
    with pytest.raises(AssertionError):
        VideoTokenizer(image_size=32, use_fsq=True, codebook_size=1024, layers=("residual",))  # M:1376
    gl = VideoTokenizer(image_size=32, codebook_size=1024, layers=("gateloop_time",))                 # M:1216-1222
    assert {"encoder_layers.0.fn.fn.norm.gamma", "encoder_layers.0.fn.fn.to_qkva.0.weight",
            "decoder_layers.0.fn.fn.to_qkva.0.weight"} <= set(gl.state_dict())
    with pytest.raises(NotImplementedError):
        VideoTokenizer(image_size=32, codebook_size=1024, dim_cond=8, layers=("cond_attend_space",))   # raises in the reference too
    with pytest.raises(AssertionError):
        VideoTokenizer(image_size=32, codebook_size=1024, layers=("cond_residual",))                   # no dim_cond (M:1151)
    with pytest.raises(TypeError):     # a plain layer after a cond layer receives cond= in the reference and fails (M:1153, M:1318)
        VideoTokenizer(image_size=32, codebook_size=1024, dim_cond=8, layers=("cond_residual", "residual"))
    m = VideoTokenizer(image_size=32, codebook_size=1024, dim_cond=8, layers=("residual", "cond_residual"))
    assert m.has_cond and m.has_cond_across_layers == [False, True]
    keys = set(m.state_dict())
    assert {"encoder_cond_in.0.weight", "decoder_cond_in.0.bias", "encoder_layers.1.to_cond.weight",
            "encoder_layers.1.conv.weights", "decoder_layers.0.conv_out.bias"} <= keys


def test_config_pickle_roundtrip_and_save_load(tmp_path):
    m = build_product(dict(image_size=32, init_dim=16, codebook_size=1024, layers=("residual", "compress_space")))
    cfg = pickle.loads(m._configs)
    assert cfg["image_size"] == 32 and cfg["layers"] == ("residual", "compress_space")
    p = tmp_path / "tok.pt"
    m.save(p)
    m2 = VideoTokenizer.init_and_load_from(p)
    for (k1, v1), (k2, v2) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2)
    m3 = copy.deepcopy(m)
    assert torch.equal(m3.conv_in.conv.weight, m.conv_in.conv.weight)


def test_load_state_dict_drops_discriminator_keys():
    m = build_product(dict(image_size=32, init_dim=16, codebook_size=1024, layers=("residual",)))
    sd = dict(m.state_dict())
    sd["discr.blocks.0.0.conv_res.weight"] = torch.zeros(3)
    m.load_state_dict(sd, strict=True)


def test_cpu_model_fails_loudly():
    """No CPU fallback: a CPU-resident model must raise, not silently run eager."""
    g = load_golden("cfg1")
    m = build_product(g["kwargs"])
    with pytest.raises(RuntimeError, match="CUDA"):
        m.tokenize(torch.randn(1, 3, 5, 32, 32))
    with pytest.raises(RuntimeError):
        m.conv_in(torch.randn(1, 3, 5, 32, 32))


def test_shape_asserts_follow_reference():
    m = build_product(dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS))
    with pytest.raises(AssertionError):
        m.tokenize(torch.randn(1, 3, 8, 32, 32))     # (8-1) % 4 != 0  (M:1691)
    with pytest.raises(AssertionError):
        m.tokenize(torch.randn(1, 3, 9, 16, 16))     # wrong image size (M:1677)
    with pytest.raises(AssertionError):
        m.decode_from_code_indices(torch.zeros(1, 3, 4, 4))   # float codes (M:1585)
    with pytest.raises(NotImplementedError):         # default ctor: use_gan=True, perceptual_loss_weight=0.1 -> GAN / VGG terms
        m(torch.randn(1, 3, 9, 32, 32), return_loss=True)
    with pytest.raises(NotImplementedError):
        m(torch.randn(1, 3, 9, 32, 32), return_discr_loss=True)
    m2 = build_product(dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS, use_gan=False,
                            perceptual_loss_weight=0.))
    with pytest.raises(RuntimeError):                # supported there, but a CPU-resident model has no kernels to run
        m2(torch.randn(1, 3, 9, 32, 32), return_loss=True)


def test_product_code_never_imports_the_oracle():
    """oracle/ is test infrastructure: the product package, the neutral data helper and bench.py's product arm must not
    import it (bench.py may, inside its CPU legs only)."""
    import ast
    import glob
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def oracle_imports(path):
        tree = ast.parse(open(path).read())
        hits = []
        for node in ast.walk(tree):
            if isinstance(node, ast.Import) and any(a.name.split(".")[0] == "oracle" for a in node.names):
                hits.append(node.lineno)
            if isinstance(node, ast.ImportFrom) and (node.module or "").split(".")[0] == "oracle":
                hits.append(node.lineno)
        return hits, tree

    for path in glob.glob(os.path.join(root, "magvit2_pytorch_b200", "*.py")) + [os.path.join(root, "synth_data.py")]:
        assert oracle_imports(path)[0] == [], path
    hits, tree = oracle_imports(os.path.join(root, "bench.py"))
    cpu_legs = {"_cpu_oracles", "run_reference_arm", "cpu_baseline_sample"}
    allowed = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in cpu_legs:
            allowed.update(range(node.lineno, node.end_lineno + 1))
    assert hits and all(h in allowed for h in hits), hits


@pytest.mark.parametrize("kt,stride", [(3, 2), (4, 2), (2, 2), (3, 1), (1, 2)])
def test_causal_conv_transpose3d_equivalent_causal_conv(kt, stride):
    """CausalConvTranspose3d (M:990-1024) = one causal conv with s * C_out channels + depth-to-time: the weight mapping the device
    path packs, checked on CPU against the reference semantics (oracle.restated.causal_conv_transpose3d)."""
    import torch.nn.functional as F
    from magvit2_pytorch_b200.modules import CausalConvTranspose3d
    from oracle.restated import causal_conv_transpose3d, causal_conv3d
    torch.manual_seed(kt * 10 + stride)
    m = CausalConvTranspose3d(5, 4, (kt, 3, 3), time_stride=stride)
    x = torch.randn(2, 5, 6, 7, 7)
    want = causal_conv_transpose3d(x, m.conv.weight.detach(), m.conv.bias.detach(), stride)
    weq, beq = m.equivalent_conv_weight()
    o = causal_conv3d(x, weq, beq)                                  # (B, (c p), T, H, W)
    b, cp, t, h, w = o.shape
    got = o.reshape(b, cp // stride, stride, t, h, w).permute(0, 1, 3, 2, 4, 5).reshape(b, cp // stride, t * stride, h, w)
    got = got[:, :, :m.output_frames(x.shape[2])]
    assert got.shape == want.shape
    assert (got - want).abs().max().item() < 1e-5
    assert set(m.state_dict()) == {"conv.weight", "conv.bias"}
    with pytest.raises(RuntimeError):
        m(x)                                                        # CPU-resident: no kernels to run, no eager fallback


def test_pack_cache_copies_and_pickles_start_empty():
    """A filled PackCache holds an engine whose ctypes handles cannot be copied: its copies and pickles are empty caches."""
    from magvit2_pytorch_b200.engine import Engine, PackCache
    c = PackCache()
    c.engine, c.packs, c._sig = Engine(None), {"w": torch.ones(2)}, ("sig", ())
    for d in (copy.copy(c), copy.deepcopy(c), pickle.loads(pickle.dumps(c))):
        assert type(d) is PackCache and (d.engine, d.packs, d._sig) == (None, None, None)
    with pytest.raises(RuntimeError):                               # bound on the module's parameters: CUDA only
        c.get(torch.nn.Linear(2, 2), "a CPU module", lambda eng: pytest.fail("packed for a CPU module"))


def test_stream_lanes_and_round_trip_refuse_cpu_models():
    """The stream front ends are CUDA-only like the model itself: a CPU-resident tokenizer is refused up front."""
    from magvit2_pytorch_b200 import HostRoundTrip, StreamLanes
    m = build_product(dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=("residual",)))
    with pytest.raises(RuntimeError):
        StreamLanes(m, 2)
    with pytest.raises(RuntimeError):
        HostRoundTrip(m, depth=2, lanes=2)
    with pytest.raises(AssertionError):
        HostRoundTrip.__init__(HostRoundTrip.__new__(HostRoundTrip), m, depth=2, lanes=3)     # more lanes than staging slots


def test_live_parameters_leave_out_what_the_reference_graph_never_reaches():
    """train.live_parameters: the dead final LayerNorm of the encoder (M:1322-1326, M:1565) and, unless
    separate_first_frame_encoding applies, the first-frame convs are not handed to the autograd Function."""
    from magvit2_pytorch_b200.train import live_parameters
    kw = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=("residual", "compress_time"))
    m = build_product(kw)
    live = {id(p) for p in live_parameters(m)}
    named = dict(m.named_parameters())
    dead = [k for k, p in named.items() if id(p) not in live]
    assert sorted(dead) == ["encoder_layers.2.1.bias", "encoder_layers.2.1.weight"]
    m2 = build_product(dict(kw, separate_first_frame_encoding=True))
    named2 = dict(m2.named_parameters())
    live_ff = {id(p) for p in live_parameters(m2, first_frame=True)}
    live_noff = {id(p) for p in live_parameters(m2, first_frame=False)}
    ff_keys = [k for k in named2 if "first_frame" in k]
    assert len(ff_keys) == 4
    assert all(id(named2[k]) in live_ff for k in ff_keys) and not any(id(named2[k]) in live_noff for k in ff_keys)
