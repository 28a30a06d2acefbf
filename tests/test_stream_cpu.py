"""Streaming tokenize / decode without a device: the chunk rule and the construction-time errors."""
import pytest
import torch

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.stream import decoder_chunk_frames, encoder_chunk_frames

KW = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024,
          layers=("residual", "compress_space", "compress_time", "residual", "compress_time"))


def test_encoder_chunk_rule():
    assert encoder_chunk_frames(1, 4, True, True) == 1
    assert encoder_chunk_frames(9, 4, True, True) == 3
    assert encoder_chunk_frames(4, 4, False, True) == 1
    assert encoder_chunk_frames(8, 4, False, False) == 2
    assert encoder_chunk_frames(8, 4, True, False) == 2
    for n, first, ff in ((4, True, True), (0, True, True), (1, False, True), (6, False, True), (0, False, True),
                         (1, True, False), (3, False, False)):
        with pytest.raises(ValueError, match="takes"):
            encoder_chunk_frames(n, 4, first, ff)


def test_decoder_chunk_rule():
    assert decoder_chunk_frames(1, 4, True, True) == 1
    assert decoder_chunk_frames(3, 4, True, True) == 9
    assert decoder_chunk_frames(1, 4, False, True) == 4
    assert decoder_chunk_frames(2, 4, True, False) == 8
    with pytest.raises(ValueError, match="at least one"):
        decoder_chunk_frames(0, 4, True, True)


@pytest.mark.parametrize("pad_mode", ["reflect", "replicate", "circular"])
def test_pad_mode_is_refused_at_construction(pad_mode):
    m = VideoTokenizer(pad_mode=pad_mode, **KW)
    with pytest.raises(NotImplementedError, match="pad_mode"):
        m.tokenize_stream(batch_size=1)
    with pytest.raises(NotImplementedError, match="pad_mode"):
        m.decode_stream(batch_size=1)


def test_construction_checks():
    m = VideoTokenizer(**KW)
    with pytest.raises(ValueError, match="batch_size"):
        m.tokenize_stream(batch_size=0)
    s = m.decode_stream(batch_size=2, video_contains_first_frame=False)
    assert s.pushes == 0 and not s.first_frame
    with pytest.raises(ValueError, match="chunk must be"):
        m.tokenize_stream(batch_size=1).push(torch.zeros(1, 3, 1, 16, 16))
