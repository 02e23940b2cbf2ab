"""matchering_b200 -- CUDA-native (H100, sm_90a) drop-in for Matchering's mastering DSP hot path.

Public surface mirrors the reference package (matchering/__init__.py:31-36):
    mg.log, mg.Result, mg.pcm16, mg.pcm24, mg.Config, mg.process, mg.load, mg.check
`process` and `stages.main` need a CUDA device and the in-tree library (python -m
matchering_b200.build); importing the package itself does not.
"""
__version__ = "0.1.0"

from .log.handlers import set_handlers as log
from .results import Result, pcm16, pcm24
from .defaults import Config, LimiterConfig
from .loader import load
from .checker import check
from .profile import ReferenceProfile, analyze_reference
from .loudness import AlbumLoudness, Loudness, album_loudness, loudness  # (the function shadows the module name on the package)


def process(*args, **kwargs):
    from .core import process as _process
    return _process(*args, **kwargs)


def process_album(*args, **kwargs):
    from .core import process_album as _process_album
    return _process_album(*args, **kwargs)


def process_versions(*args, **kwargs):
    from .core import process_versions as _process_versions
    return _process_versions(*args, **kwargs)
