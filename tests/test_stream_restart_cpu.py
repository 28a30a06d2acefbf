"""Restarting single rows of a stream without a device: the argument checks of restart() and the host arithmetic of the
time attention's per-row key starts (engine.row_runs, engine.kv_cache_plan, StreamState.restart_rows)."""
import pytest
import torch

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.engine import StreamState, kv_cache_plan, row_runs
from magvit2_pytorch_b200.stream import restart_rows

KW = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024,
          layers=("residual", "compress_space", "compress_time", "residual", "compress_time"))
COND_KW = dict(KW, dim_cond=12, layers=("residual", "compress_space", "compress_time", "cond_residual"))


def _streams(m, **kw):
    return m.tokenize_stream(**kw), m.decode_stream(**kw)


def test_rows_argument():
    assert restart_rows([2, 0], 3) == [2, 0]
    assert restart_rows(torch.tensor([1]), 3) == [1]
    assert restart_rows(torch.tensor([], dtype=torch.long), 3) == []
    assert restart_rows((), 3) == []
    for bad, match in (([3], "lie in"), ([-1], "lie in"), ([1, 1], "distinct"), (torch.tensor([0, 0]), "distinct"),
                       ([0.0], "integers"), ([True], "integers"), (torch.tensor([0.0]), "1-D integer"),
                       (torch.tensor([[0]]), "1-D integer"), (torch.tensor([True]), "1-D integer")):
        with pytest.raises(ValueError, match=match):
            restart_rows(bad, 3)


@pytest.mark.parametrize("which", [0, 1])
def test_restart_refuses_bad_rows(which):
    s = _streams(VideoTokenizer(**KW), batch_size=3)[which]
    for rows in ([3], [0, 0], [-1]):
        with pytest.raises(ValueError, match="rows"):
            s.restart(rows)
    s.restart([0, 2])                                   # before the first push: nothing to reset
    assert s.pushes == 0 and not s._restarted


@pytest.mark.parametrize("which", [0, 1])
def test_restart_checks_cond(which):
    m = VideoTokenizer(**COND_KW)
    cond = torch.randn(3, 12)
    s = _streams(m, batch_size=3, cond=cond)[which]
    assert s.cond is not cond and torch.equal(s.cond, cond)
    for bad in (None, torch.randn(1, 12), torch.randn(2, 11), torch.randn(2), torch.zeros(2, 12, dtype=torch.long),
                [[0.0] * 12] * 2):
        with pytest.raises(ValueError, match="cond"):
            s.restart([0, 1], cond=bad)
    assert torch.equal(s.cond, cond)                    # a refused restart changes nothing
    new = torch.randn(2, 12, dtype=torch.float64)
    keep = new.clone()
    s.restart([2, 0], cond=new)
    assert torch.equal(new, keep)                       # the caller's tensor is not touched
    assert torch.equal(s.cond[1], cond[1])
    assert torch.equal(s.cond[[2, 0]], new.float())
    cond.zero_()                                        # the stream holds its own copy
    assert torch.equal(s.cond[[2, 0]], new.float())


def test_restart_refuses_separate_first_frame_encoding():
    m = VideoTokenizer(separate_first_frame_encoding=True, **KW)
    for s in _streams(m, batch_size=2):
        with pytest.raises(NotImplementedError, match="separate_first_frame_encoding"):
            s.restart([0])
    for s in _streams(m, batch_size=2, video_contains_first_frame=False):
        s.restart([0])


def test_row_runs():
    assert row_runs([0, 0, 0]) == [(0, 3, 0)]
    assert row_runs([0, 5, 5, 0]) == [(0, 1, 0), (1, 3, 5), (3, 4, 0)]
    assert row_runs([3]) == [(0, 1, 3)]
    assert row_runs([False, True, True]) == [(0, 1, False), (1, 3, True)]


def test_kv_cache_plan():
    # no restart: every row starts at 0, nothing is dropped and the cache grows by the step, as before restarts existed
    assert kv_cache_plan(16, 1, (0, 0), 16) == (0, 32)
    assert kv_cache_plan(0, 3, (0, 0), 16) == (0, 16)
    # the earliest live clip starts at 9: frames 0..8 go, 7 + 1 frames fit in one step
    assert kv_cache_plan(16, 1, (9, 12, 15, 10), 16) == (9, 16)
    # every row restarted at the end of the cache: all of it goes
    assert kv_cache_plan(16, 2, (16, 16), 16) == (16, 16)
    assert kv_cache_plan(32, 4, (3, 20), 16) == (3, 48)


def test_restart_rows_resets_the_carried_state():
    B = 3
    ss = StreamState()
    hist = torch.ones(B, 2, 2, 2, 4)
    prev = torch.ones(B, 1, 2, 2, 4)
    scan = torch.ones(B, 4, 4)
    kv = torch.ones(B, 16, 2, 2, 8)
    a = ss.sub("enc0").sub("conv3")
    a.put("hist", (hist, 2))
    b = ss.sub("enc1").sub("attn")
    b.put("prev", prev)
    b.put("kv", (kv, 7, (0, 0, 0)))
    ss.sub("enc2").put("s", scan)
    counts = ss.history_counts()
    ss.restart_rows([0, 2])
    for t in (hist, prev, scan):
        assert t[0].eq(0).all() and t[2].eq(0).all() and t[1].eq(1).all()
    assert kv.eq(1).all()                               # the keys stay; the rows' starts move to the end of the cache
    assert b.get("kv")[0] is kv and b.get("kv")[1:] == (7, (7, 0, 7))
    assert ss.history_counts() == counts and ss.kv_capacities() == (16,)
