"""mg.process (reference: matchering/core.py:32-121): files in, mastered files out.  Loading,
validation and saving are host plumbing; `stages.main` in the middle runs on the GPU."""
from .checker import check, check_equality
from .defaults import Config
from .loader import load
from .log import Code, ModuleError, debug, debug_enabled, debug_line, info
from .profile import ReferenceProfile
from .results import Result
from .saver import save
from .stages import main_device
from .utils import get_temp_folder

_DEFAULT_CONFIG = None


def process(target: str, reference, results: list, config: Config = None,
            preview_target: Result = None, preview_result: Result = None):
    """`reference` is a file path or a ReferenceProfile (mg.analyze_reference): mastering many targets against
    one reference analyses it once.  With a profile the allow_equality check has no reference samples to
    compare with and is skipped."""
    global _DEFAULT_CONFIG
    if config is None:
        if _DEFAULT_CONFIG is None:
            _DEFAULT_CONFIG = Config()
        config = _DEFAULT_CONFIG
    debug_line()
    info(Code.INFO_LOADING)
    if not results:
        raise RuntimeError("The result list is empty")
    temp_folder = config.temp_folder if config.temp_folder else get_temp_folder(results)

    # native_rate: the target as loaded (stereo, at its own rate), for stages 2-4 when that rate is not the internal one
    native_audio, native_rate = None, config.internal_sample_rate
    if isinstance(reference, ReferenceProfile):
        # the reference was loaded, checked and analysed when the profile was made; only its fingerprint is
        # compared with this Config here.  There are no reference samples to compare the target with.
        reference.check_config(config)
        target_audio, target_rate, native_audio, native_rate = _load_and_check_target(target, temp_folder, config)
        if not config.allow_equality:
            debug("The REFERENCE is a profile: the check that the TARGET differs from it is skipped")
        if (target_rate != config.internal_sample_rate or target_audio.shape[1] != 2
                or not target_audio.shape[0] > config.fft_size):
            raise ModuleError(Code.ERROR_VALIDATION)
        reference_audio = reference
    else:
        target_audio, target_rate, native_audio, native_rate = _load_and_check_target(target, temp_folder, config)
        reference_audio, reference_rate = _load_and_check(reference, "reference", temp_folder, config)
        if not config.allow_equality:
            _check_equality_any(target_audio, reference_audio)
        if (not (target_rate == reference_rate == config.internal_sample_rate)
                or not (target_audio.shape[1] == reference_audio.shape[1] == 2)
                or not (target_audio.shape[0] > config.fft_size and reference_audio.shape[0] > config.fft_size)):
            raise ModuleError(Code.ERROR_VALIDATION)

    needs = dict(need_default=any(r.use_limiter for r in results),
                 need_no_limiter=any(not r.use_limiter and not r.normalize for r in results),
                 need_no_limiter_normalized=any(not r.use_limiter and r.normalize for r in results))
    if native_rate != config.internal_sample_rate:
        from .plan import native_config
        from .stages import main_native_device
        limited, plain, normalized = main_native_device(native_audio, native_rate, reference_audio, config,
                                                        analysis=target_audio, **needs)
        # results and previews at the target's rate: the preview windows keep their length in seconds
        out_config, preview_source = native_config(config, native_rate), native_audio
    else:
        limited, plain, normalized = main_device(target_audio, reference_audio, config, **needs)
        out_config, preview_source = config, target_audio

    debug_line()
    info(Code.INFO_EXPORTING)
    for wanted in results:
        audio = limited if wanted.use_limiter else (normalized if wanted.normalize else plain)
        _export(wanted, audio, out_config.internal_sample_rate)
    if preview_target or preview_result:
        from .preview_creator import create_preview
        first = next(item for item in (limited, plain, normalized) if item is not None)
        create_preview(preview_source, first, out_config, preview_target, preview_result)
    debug_line()
    info(Code.INFO_COMPLETED)


def process_album(targets: list, reference, results: list, config: Config = None, album_loudness_target: float = None):
    """Master an album: `targets` is a list of file paths, `results` a list of the same length whose entries are lists
    of Result as mg.process takes them.  Every target is loaded and checked as mg.process loads its target; then ONE
    level match and ONE matching FIR, from statistics pooled over every track (stages.main_album), master them all, so
    the tracks keep their relative levels.  `reference` is a file path or a ReferenceProfile.  Config(loudness_target=...)
    and native-rate targets are refused.  album_loudness_target (LUFS): the limited results are driven with ONE limiter
    gain until the album, metered as one programme (mg.album_loudness), reads that loudness."""
    from .stages import album_check, main_album_device
    if config is None:
        config = Config()
    targets, results = list(targets), list(results)
    if not targets or len(targets) != len(results):
        raise ValueError(f"process_album: {len(targets)} targets and {len(results)} result lists")
    album_check(len(targets), config, album_loudness_target)
    if any(not r for r in results):
        raise ValueError("process_album: every track needs at least one Result")
    if config.native_rate:
        for t in targets:
            rate = _file_rate(t)
            if rate is not None and rate != config.internal_sample_rate:
                raise ValueError(f"process_album: '{t}' is at {rate} Hz; albums are mastered at the internal rate "
                                 f"({config.internal_sample_rate} Hz), not at native rates")
    debug_line()
    info(Code.INFO_LOADING)
    temp_folder = config.temp_folder if config.temp_folder else get_temp_folder([r for rs in results for r in rs])
    reference_audio = None
    if isinstance(reference, ReferenceProfile):
        reference.check_config(config)
    else:
        reference_audio, reference_rate = _load_and_check(reference, "reference", temp_folder, config)
        if (reference_rate != config.internal_sample_rate or reference_audio.shape[1] != 2
                or not reference_audio.shape[0] > config.fft_size):
            raise ModuleError(Code.ERROR_VALIDATION)
    audios = []
    for t in targets:
        audio, rate, _, native_rate = _load_and_check_target(t, temp_folder, config)
        if native_rate != config.internal_sample_rate:
            raise ValueError(f"process_album: '{t}' is at {native_rate} Hz; albums are mastered at the internal rate")
        if reference_audio is not None and not config.allow_equality:
            _check_equality_any(audio, reference_audio)
        if rate != config.internal_sample_rate or audio.shape[1] != 2 or not audio.shape[0] > config.fft_size:
            raise ModuleError(Code.ERROR_VALIDATION)
        audios.append(audio)
    if reference_audio is not None:
        from .profile import analyze_reference
        reference = analyze_reference(reference_audio, config)

    everything = [r for rs in results for r in rs]
    needs = dict(need_default=any(r.use_limiter for r in everything),
                 need_no_limiter=any(not r.use_limiter and not r.normalize for r in everything),
                 need_no_limiter_normalized=any(not r.use_limiter and r.normalize for r in everything))
    outs = main_album_device(audios, reference, config, album_loudness_target=album_loudness_target, **needs)
    if album_loudness_target is not None and needs["need_default"] and debug_enabled():
        from .loudness import album_loudness
        m = album_loudness([limited for limited, _, _ in outs], config.internal_sample_rate)
        debug(f"The album's masters read {m.album.integrated:.4f} LUFS as one programme")
        for t, (path, track) in enumerate(zip(targets, m.tracks)):
            debug(f"Master {t + 1} ('{path}'): {track.integrated:.4f} LUFS, true peak {track.true_peak:.2f} dBTP")
    debug_line()
    info(Code.INFO_EXPORTING)
    for (limited, plain, normalized), wanted_list in zip(outs, results):
        for wanted in wanted_list:
            audio = limited if wanted.use_limiter else (normalized if wanted.normalize else plain)
            _export(wanted, audio, config.internal_sample_rate)
    debug_line()
    info(Code.INFO_COMPLETED)


def process_versions(targets: list, reference, results: list, config: Config = None):
    """Master a mix and its versions as linked versions (stages.main_versions): `targets[0]` is the main mix's file,
    the others its versions' (instrumental, a cappella, TV mix, clean edit), all of one length and one sample rate;
    `results` holds a list of Result per target, as mg.process takes them.  Every file is loaded and checked as
    mg.process loads its target.  The versions take the main's match and the main's limiter gain, so that every
    master nulls against the main's: main master - instrumental master is the vocal through the same chain.
    `reference` is a file path or a ReferenceProfile.  Versions of another length or rate, more than 8 versions and
    native-rate targets off the internal rate are refused before any device work."""
    from ._native import MGB_MAX_VERSIONS
    from .stages import main_versions_device, versions_check
    if config is None:
        config = Config()
    targets, results = list(targets), list(results)
    if not targets or len(targets) != len(results):
        raise ValueError(f"process_versions: {len(targets)} targets and {len(results)} result lists")
    if len(targets) - 1 > MGB_MAX_VERSIONS:
        raise ValueError(f"process_versions: {len(targets) - 1} versions, at most {MGB_MAX_VERSIONS}")
    if any(not r for r in results):
        raise ValueError("process_versions: every target needs at least one Result")
    rates = [_file_rate(t) for t in targets]
    if config.native_rate:
        for t, rate in zip(targets, rates):
            if rate is not None and rate != config.internal_sample_rate:
                raise ValueError(f"process_versions: '{t}' is at {rate} Hz; versions are mastered at the internal rate "
                                 f"({config.internal_sample_rate} Hz), not at native rates")
    for t, rate in zip(targets[1:], rates[1:]):
        if rate is not None and rates[0] is not None and rate != rates[0]:
            raise ValueError(f"process_versions: '{t}' is at {rate} Hz, the main mix at {rates[0]} Hz")
    debug_line()
    info(Code.INFO_LOADING)
    temp_folder = config.temp_folder if config.temp_folder else get_temp_folder([r for rs in results for r in rs])
    reference_audio = None
    if isinstance(reference, ReferenceProfile):
        reference.check_config(config)
    else:
        reference_audio, reference_rate = _load_and_check(reference, "reference", temp_folder, config)
        if (reference_rate != config.internal_sample_rate or reference_audio.shape[1] != 2
                or not reference_audio.shape[0] > config.fft_size):
            raise ModuleError(Code.ERROR_VALIDATION)
    audios = []
    for t in targets:
        audio, rate, _, native_rate = _load_and_check_target(t, temp_folder, config)
        if native_rate != config.internal_sample_rate:
            raise ValueError(f"process_versions: '{t}' is at {native_rate} Hz; versions are mastered at the internal rate")
        if reference_audio is not None and not config.allow_equality:
            _check_equality_any(audio, reference_audio)
        if rate != config.internal_sample_rate or audio.shape[1] != 2 or not audio.shape[0] > config.fft_size:
            raise ModuleError(Code.ERROR_VALIDATION)
        audios.append(audio)
    versions_check(audios, config)

    everything = [r for rs in results for r in rs]
    needs = dict(need_default=any(r.use_limiter for r in everything),
                 need_no_limiter=any(not r.use_limiter and not r.normalize for r in everything),
                 need_no_limiter_normalized=any(not r.use_limiter and r.normalize for r in everything))
    outs = main_versions_device(audios, reference if reference_audio is None else reference_audio, config, **needs)
    debug_line()
    info(Code.INFO_EXPORTING)
    for (limited, plain, normalized), wanted_list in zip(outs, results):
        for wanted in wanted_list:
            audio = limited if wanted.use_limiter else (normalized if wanted.normalize else plain)
            _export(wanted, audio, config.internal_sample_rate)
    debug_line()
    info(Code.INFO_COMPLETED)


def _file_rate(path) -> int | None:
    """The sample rate a file's header states, or None when it cannot be read without decoding."""
    from . import wavio
    from .results import real_soundfile
    try:
        with open(path, "rb") as f:
            layout = wavio._pcm_layout(f)
        if layout is not None:
            return layout[2]
        sf = real_soundfile()
        return int(sf.info(path).samplerate) if sf is not None else None
    except (OSError, RuntimeError):
        return None


def _export(wanted: Result, audio, sample_rate: int, name: str = "result") -> None:
    """16/24-bit WAV results are quantised on the device and written as they come back (a quarter of
    the device->host bytes of a float64 array); everything else takes the reference's route through
    a host float array and `save`.  Dithered results (Result(dither=...)) are always quantised on the device,
    by the dithered encoder, whether or not libsndfile is present."""
    from .results import real_soundfile
    is_wav = wanted.file.lower().endswith(".wav")
    dither = getattr(wanted, "dither", None)
    if is_wav and wanted.subtype in ("PCM_16", "PCM_24") and (dither is not None or real_soundfile() is None):
        from . import wavio
        from .engine import encode_pcm
        bits = int(wanted.subtype[4:])
        params = None
        if dither is not None:
            from .dither import params as dither_params
            params = dither_params(dither, sample_rate, wanted.dither_seed)
            debug(f"Dither: {dither}, seed {wanted.dither_seed}")
        debug(f"Saving the {name.upper()} {sample_rate} Hz Stereo {wanted.subtype} to: '{wanted.file}'...")
        wavio.write_pcm(wanted.file, encode_pcm(audio, bits, params), sample_rate, bits)
        debug(f"'{wanted.file}' is saved")
    else:
        save(wanted.file, audio.cpu().numpy().astype("float64"), sample_rate, wanted.subtype, name)


def _load_and_check(file: str, name: str, temp_folder: str, config: Config):
    """16/24-bit PCM WAV at the internal rate is decoded and checked on the device; everything else
    goes through the host loader and checker like in the reference."""
    from .device_io import check_on_device, load_to_device
    on_device = load_to_device(file, name, config)
    if on_device is not None:
        audio, rate = on_device
        return check_on_device(audio, config, name, rate), config.internal_sample_rate
    audio, rate = load(file, name, temp_folder)
    return check(audio, rate, config, name)


def _load_and_check_target(file: str, temp_folder: str, config: Config):
    """-> (the target at the internal rate, that rate, the target as loaded in stereo or None, its rate).  The
    loaded copy is kept only for Config(native_rate=True)."""
    if not config.native_rate:
        audio, rate = _load_and_check(file, "target", temp_folder, config)
        return audio, rate, None, rate
    from .device_io import check_on_device, load_to_device
    on_device = load_to_device(file, "target", config)
    if on_device is not None:
        audio, rate = on_device
        audio, native = check_on_device(audio, config, "target", rate, native=True)
        return audio, config.internal_sample_rate, native, rate
    audio, rate = load(file, "target", temp_folder)
    checked, checked_rate, native = check(audio, rate, config, "target", native=True)
    return checked, checked_rate, native, rate


def _check_equality_any(target_audio, reference_audio) -> None:
    import torch
    if isinstance(target_audio, torch.Tensor) and isinstance(reference_audio, torch.Tensor):
        from .device_io import check_equality_on_device
        check_equality_on_device(target_audio, reference_audio)
    else:
        as_np = lambda a: a.cpu().numpy() if isinstance(a, torch.Tensor) else a
        check_equality(as_np(target_audio), as_np(reference_audio))
