"""magvit2_pytorch_b200 -- H100-native (sm_90a) VideoTokenizer forward path.

Drop-in for ``magvit2_pytorch.VideoTokenizer`` inference (tokenize / decode_from_code_indices /
forward) behind the C ABI of libmagvit2_b200.so.  See DESIGN.md / INTEGRATION.md.
"""
from .video_tokenizer import VideoTokenizer, __version__  # noqa: F401
from .host_io import HostRoundTrip, StreamLanes  # noqa: F401
from .modules import CausalConvTranspose3d  # noqa: F401
from .stream import DecodeStream, TokenizeStream  # noqa: F401
from . import _lib  # noqa: F401

__all__ = ["VideoTokenizer", "HostRoundTrip", "StreamLanes", "CausalConvTranspose3d", "TokenizeStream", "DecodeStream"]
