"""Result descriptors (reference: matchering/results.py:25-46).  The reference validates
(extension, subtype) through libsndfile; this build writes WAV itself (saver.py) and accepts the
WAV subtypes it can encode -- anything else raises TypeError exactly where the reference would
for a format libsndfile does not know."""
import os

WAV_SUBTYPES = ("PCM_16", "PCM_24", "PCM_32", "FLOAT", "DOUBLE")
_FORMATS = {"WAV": WAV_SUBTYPES}


def real_soundfile():
    """libsndfile's binding when it is really installed (not a test stand-in), else None."""
    try:
        import soundfile as sf
    except ImportError:
        return None
    return sf if getattr(sf, "__libsndfile_version__", None) else None


def _check_format(ext: str, subtype: str = None) -> bool:
    sf = real_soundfile()  # used when present, so FLAC/AIFF/... keep working
    if sf is not None:
        return bool(sf.check_format(ext, subtype))
    if ext not in _FORMATS:
        return False
    return subtype is None or subtype in _FORMATS[ext]


class Result:
    """dither: None (plain rounding, libsndfile's), "tpdf" (flat TPDF dither) or "shaped" (TPDF dither, noise-shaped
    by dither.shaping_filter at the Config's internal rate), for 16- and 24-bit WAV results only; dither_seed selects
    the dither's noise (the same seed gives the same file)."""

    def __init__(self, file: str, subtype: str, use_limiter: bool = True, normalize: bool = True, dither: str = None,
                 dither_seed: int = 0):
        ext = os.path.splitext(file)[1][1:].upper()
        if not _check_format(ext):
            raise TypeError(f"{ext} format is not supported")
        if not _check_format(ext, subtype):
            raise TypeError(f"{ext} format does not have {subtype} subtype")
        if dither is not None:
            from .dither import check_kind
            check_kind(dither)
            if ext != "WAV" or subtype not in ("PCM_16", "PCM_24"):
                raise ValueError(f"dither applies to 16- and 24-bit WAV results, not {ext} {subtype}")
            if isinstance(dither_seed, bool) or not isinstance(dither_seed, int) or not 0 <= dither_seed < 2 ** 64:
                raise ValueError(f"dither_seed must be an integer in [0, 2^64), not {dither_seed!r}")
        self.file = file
        self.subtype = subtype
        self.use_limiter = use_limiter
        self.normalize = normalize
        self.dither = dither
        self.dither_seed = dither_seed


def pcm16(file: str, dither: str = None, dither_seed: int = 0) -> Result:
    return Result(file, "PCM_16", dither=dither, dither_seed=dither_seed)


def pcm24(file: str, dither: str = None, dither_seed: int = 0) -> Result:
    return Result(file, "PCM_24", dither=dither, dither_seed=dither_seed)
