"""GPU drop-in for matchering/stages.py: same `main` signature and returns (stages.py:210-272),
same four stages and the same info codes between them; every array operation runs in
libmatchering_b200 on the current CUDA device."""
from __future__ import annotations

import math

import torch

from . import _native, plan as _plan
from .defaults import Config
from .engine import (TrackSession, album_finalize_to_loudness, album_match, get_native_plan, get_plan, host_array_ok, stages_main_host,
                     stages_main_host_profiled, to_device_f32, to_host_like, versions_finalize, versions_match)
from .log import Code, info, debug, debug_line, debug_enabled
from .profile import ReferenceProfile
from .utils import to_db


def main(target, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
         need_no_limiter_normalized: bool = False):
    """target, reference: (N, 2) stereo at config.internal_sample_rate, numpy (float64 like the
    reference's loader produces, or float32) or torch tensors.  Returns
    (result, result_no_limiter, result_no_limiter_normalized), None where not requested, in the
    caller's array type.  `reference` may also be a ReferenceProfile (profile.analyze_reference): the
    level statistics and FIR are bit-identical to passing the samples it was made from, and no reference bytes
    are moved.

    numpy in -> the whole job is ONE native call (mgb_stages_main_host): the library narrows and uploads
    the caller's pageable arrays chunk by chunk on its own worker threads, runs the four stages and
    returns float64 (or float32) arrays DMA'd into pooled pinned memory.  torch in -> the staged path
    below, results stay on the device."""
    profiled = isinstance(reference, ReferenceProfile)
    if profiled:
        reference.check_config(config)
    # (a loudness target runs its search in the device session below; the single-call host entry has no target)
    if host_array_ok(target) and (profiled or host_array_ok(reference)) and config.loudness_target is None:
        plan = get_plan(config)
        with torch.cuda.device(plan.device):
            debug_line()
            info(Code.INFO_MATCHING_LEVELS)          # stages.py:52
            debug(f"The maximum size of the analyzed piece: {config.max_piece_size} samples "
                  f"or {config.max_piece_size / config.internal_sample_rate:.2f} seconds")
            info(Code.INFO_MATCHING_FREQS)           # stages.py:117
            info(Code.INFO_CORRECTING_LEVELS)        # stages.py:147
            info(Code.INFO_FINALIZING)               # stages.py:182
            if profiled:
                outs, st = stages_main_host_profiled(plan, target, reference, need_default, need_no_limiter,
                                                     need_no_limiter_normalized)
            else:
                outs, st = stages_main_host(plan, target, reference, need_default, need_no_limiter,
                                            need_no_limiter_normalized)
            if debug_enabled():
                L = (plan.layout_profiled(target.shape[0]) if profiled
                     else plan.layout(target.shape[0], reference.shape[0]))
                _debug_scalars(st, L, reference if profiled else None)
        return outs
    outs = main_device(target, reference, config, need_default, need_no_limiter, need_no_limiter_normalized)
    return tuple(None if t is None else to_host_like(t, target) for t in outs)


def _debug_scalars(st, L, profile: ReferenceProfile | None = None) -> None:
    debug(f"The TARGET will be didived into {L.target_divisions} pieces of {L.target_piece} samples; "
          f"{st.target_loud_pieces} of them are at least as loud as the average")
    # a profiled layout has no reference pieces of its own: the profile recorded the reference's geometry
    divisions, piece = (profile.divisions, profile.piece) if profile is not None else (L.reference_divisions,
                                                                                        L.reference_piece)
    debug(f"The REFERENCE will be didived into {divisions} pieces of {piece} samples; "
          f"{st.reference_loud_pieces} of them are at least as loud as the average")
    if st.final_amplitude_coef != 1.0:
        debug(f"The REFERENCE was normalized. Final amplitude coefficient for the TARGET audio is: "
              f"{to_db(st.final_amplitude_coef)}")
    debug(f"The RMS coefficient is: {to_db(st.rms_coefficient)}")
    for step in range(st.steps_done):
        debug(f"RMS correction #{step + 1}: {to_db(st.correction[step])}")
    debug("The limiter is not needed!" if not st.limiter_engaged else "The limiter was applied")


def main_device(target, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
                need_no_limiter_normalized: bool = False):
    """Same as `main`, but the results stay on the device as float32 CUDA tensors (the caller may
    quantise them there, see core.process).  `reference` may be a ReferenceProfile."""
    profiled = isinstance(reference, ReferenceProfile)
    if profiled:
        reference.check_config(config)
    plan = get_plan(config)
    device = plan.device
    if target.ndim != 2 or target.shape[1] != 2 or (not profiled and (reference.ndim != 2 or reference.shape[1] != 2)):
        raise ValueError("target and reference must be (frames, 2) stereo arrays")
    with torch.cuda.device(device):
        d_target = to_device_f32(target, device)
        if profiled:
            d_profile = reference.checked_blob(plan)
            session = TrackSession(plan, d_target.shape[0], None)
        else:
            d_reference = to_device_f32(reference, device)
            session = TrackSession(plan, d_target.shape[0], d_reference.shape[0])

        debug_line()
        info(Code.INFO_MATCHING_LEVELS)          # stages.py:52
        debug(f"The maximum size of the analyzed piece: {config.max_piece_size} samples "
              f"or {config.max_piece_size / config.internal_sample_rate:.2f} seconds")
        if profiled:
            session.match_levels_profiled(d_target, d_profile)
        else:
            session.match_levels(d_target, d_reference)

        debug_line()
        info(Code.INFO_MATCHING_FREQS)           # stages.py:117
        session.match_frequencies(d_target)

        debug_line()
        info(Code.INFO_CORRECTING_LEVELS)        # stages.py:147
        session.correct_levels()

        debug_line()
        info(Code.INFO_FINALIZING)               # stages.py:182
        report = None
        if need_default and config.loudness_target is not None:
            limited, plain, normalized, report = session.finalize_to_loudness(config.loudness_target, need_no_limiter,
                                                                              need_no_limiter_normalized)
        else:
            limited, plain, normalized = session.finalize(need_default, need_no_limiter, need_no_limiter_normalized)

        if debug_enabled():  # one read-back of the device scalars, only when somebody listens
            _debug_scalars(session.read_state(), session.layout, reference if profiled else None)
            if report is not None:
                from .loudness import LoudnessTarget, debug_target
                raw = report.cpu().numpy().tobytes()
                debug_target(LoudnessTarget.from_report(config.loudness_target,
                                                        _native.LoudnessTargetReport.from_buffer_copy(raw)))

    return limited, plain, normalized


def main_native(target, sample_rate: int, reference, config: Config, need_default: bool = True,
                need_no_limiter: bool = False, need_no_limiter_normalized: bool = False):
    """`main` for a target at its own rate `sample_rate` (DESIGN.md section 4 "Native-rate masters"): the level and
    spectrum match is analysed on the target resampled to config.internal_sample_rate, as `main` would see it, and the
    FIR, the RMS correction, the limiter (true peak, loudness target) then run on the target's own samples, so every
    output is at `sample_rate` with the target's length.  target: (N, 2) or mono (N, 1), numpy or torch; the outputs
    come back in its array type.  At sample_rate == internal_sample_rate this is `main`."""
    if int(sample_rate) == config.internal_sample_rate:
        return main(target, reference, config, need_default, need_no_limiter, need_no_limiter_normalized)
    outs = main_native_device(target, sample_rate, reference, config, need_default, need_no_limiter,
                              need_no_limiter_normalized)
    return tuple(None if t is None else to_host_like(t, target) for t in outs)


def main_native_device(target, sample_rate: int, reference, config: Config, need_default: bool = True,
                       need_no_limiter: bool = False, need_no_limiter_normalized: bool = False, analysis=None):
    """`main_native` with the results left on the device as float32 CUDA tensors.  `analysis`: the target already
    resampled to the internal rate (mg.process's loaders make it while checking the target); made here otherwise."""
    sample_rate = int(sample_rate)
    if sample_rate == config.internal_sample_rate:
        return main_device(target, reference, config, need_default, need_no_limiter, need_no_limiter_normalized)
    profiled = isinstance(reference, ReferenceProfile)
    if profiled:
        reference.check_config(config)
    if target.ndim != 2 or target.shape[1] not in (1, 2) or (not profiled and (reference.ndim != 2 or reference.shape[1] != 2)):
        raise ValueError("the target must be (frames, 2) or (frames, 1) and the reference (frames, 2)")
    _plan.native_check_length(config, sample_rate, int(target.shape[0]))  # (raises before any device work)
    plan = get_plan(config)
    nplan = get_native_plan(config, sample_rate, plan.device)
    device = plan.device
    with torch.cuda.device(device):
        d_native = to_device_f32(target, device)
        if d_native.shape[1] == 1:
            d_native = d_native.repeat(1, 2).contiguous()
        if analysis is None:
            from .resample import resample_on_device
            d_target = resample_on_device(d_native, sample_rate, config.internal_sample_rate)
        else:
            d_target = to_device_f32(analysis, device)
        if profiled:
            d_profile = reference.checked_blob(plan)
            session = TrackSession(plan, d_target.shape[0], None)
        else:
            d_reference = to_device_f32(reference, device)
            session = TrackSession(plan, d_target.shape[0], d_reference.shape[0])
        native = TrackSession(nplan, d_native.shape[0], None)

        debug_line()
        info(Code.INFO_MATCHING_LEVELS)          # stages.py:52
        debug(f"The maximum size of the analyzed piece: {config.max_piece_size} samples "
              f"or {config.max_piece_size / config.internal_sample_rate:.2f} seconds")
        if profiled:
            session.match_levels_profiled(d_target, d_profile)
        else:
            session.match_levels(d_target, d_reference)

        debug_line()
        info(Code.INFO_MATCHING_FREQS)           # stages.py:117
        debug(f"The FIR is designed at {config.internal_sample_rate} Hz and applied at {sample_rate} Hz "
              f"({nplan.tables.fft_size} points)")
        session.design_frequencies()
        native.match_frequencies_native(session, d_native)

        debug_line()
        info(Code.INFO_CORRECTING_LEVELS)        # stages.py:147
        native.correct_levels()

        debug_line()
        info(Code.INFO_FINALIZING)               # stages.py:182
        report = None
        if need_default and config.loudness_target is not None:
            limited, plain, normalized, report = native.finalize_to_loudness(config.loudness_target, need_no_limiter,
                                                                             need_no_limiter_normalized)
        else:
            limited, plain, normalized = native.finalize(need_default, need_no_limiter, need_no_limiter_normalized)

        if debug_enabled():
            _debug_scalars(native.read_state(), session.layout, reference if profiled else None)
            if report is not None:
                from .loudness import LoudnessTarget, debug_target
                raw = report.cpu().numpy().tobytes()
                debug_target(LoudnessTarget.from_report(config.loudness_target,
                                                        _native.LoudnessTargetReport.from_buffer_copy(raw)))

    return limited, plain, normalized


def main_album(targets, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
               need_no_limiter_normalized: bool = False, album_loudness_target: float | None = None):
    """Master the K tracks of an album against one reference with ONE level match and ONE matching FIR, from
    statistics pooled over every piece of every track (DESIGN.md section 4 "Album mastering"), so the tracks keep their
    relative levels and share one tonal correction.  targets: a list of (N_t, 2) stereo arrays at
    config.internal_sample_rate, numpy or torch; reference: samples or a ReferenceProfile.  Returns one
    (result, result_no_limiter, result_no_limiter_normalized) per track, None where not requested, in each target's
    array type.  The normalized result is normalised per track, as in `main`.  A one-track album is `main` with the
    reference's profile, bit for bit.

    album_loudness_target (LUFS): drive every track's limiter with ONE gain, searched until the album, metered as one
    programme (mg.album_loudness), reads that integrated loudness (DESIGN.md section 4 "Album loudness").  Where no
    limiter engages every track gets the same gain, so the relative levels hold exactly.  Only the limited results
    are targeted."""
    outs = main_album_device(targets, reference, config, need_default, need_no_limiter, need_no_limiter_normalized,
                             album_loudness_target=album_loudness_target)
    return [tuple(None if t is None else to_host_like(t, target) for t in track) for track, target in zip(outs, targets)]


def album_check(count: int, config: Config, album_loudness_target=None) -> None:
    """The album requests main_album refuses before any device work."""
    if album_loudness_target is not None and not (
            isinstance(album_loudness_target, (int, float)) and not isinstance(album_loudness_target, bool)
            and math.isfinite(album_loudness_target) and -70 < album_loudness_target < 0):
        raise ValueError("album_loudness_target must be None or a finite LUFS value in (-70, 0)")
    if count < 1:
        raise ValueError("an album needs at least one track")
    if count > _native.MGB_MAX_ALBUM_TRACKS:
        raise ValueError(f"an album of {count} tracks: at most {_native.MGB_MAX_ALBUM_TRACKS} are mastered together")
    if config.loudness_target is not None:
        raise ValueError("Config(loudness_target=...) is not available for albums: a target per track would undo the "
                         "album's level relation; album_loudness_target=... drives the whole album with one gain")


def main_album_device(targets, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
                      need_no_limiter_normalized: bool = False, fir_out=None, album_loudness_target: float | None = None):
    """`main_album` with the results left on the device as float32 CUDA tensors.  fir_out: optional (2, fft_size)
    float64 CUDA tensor that receives the album's mid and side FIRs."""
    targets = list(targets)
    album_check(len(targets), config, album_loudness_target)
    for target in targets:
        if target.ndim != 2 or target.shape[1] != 2:
            raise ValueError("every target must be a (frames, 2) stereo array")
        if not target.shape[0] > config.fft_size:
            raise ValueError(f"every target must be longer than fft_size ({config.fft_size} frames)")
    if not isinstance(reference, ReferenceProfile):
        from .profile import analyze_reference
        reference = analyze_reference(reference, config)
    reference.check_config(config)
    plan = get_plan(config)
    device = plan.device
    with torch.cuda.device(device):
        d_profile = reference.checked_blob(plan)
        d_targets = [to_device_f32(t, device) for t in targets]
        sessions = [TrackSession(plan, int(t.shape[0]), None) for t in d_targets]

        debug_line()
        info(Code.INFO_MATCHING_LEVELS)
        debug(f"Album of {len(sessions)} tracks, pieces per track: {[int(s.layout.target_divisions) for s in sessions]}")
        info(Code.INFO_MATCHING_FREQS)
        info(Code.INFO_CORRECTING_LEVELS)
        album_match(sessions, d_targets, d_profile, fir_out)

        debug_line()
        info(Code.INFO_FINALIZING)
        report = None
        if need_default and album_loudness_target is not None:
            outs, report = album_finalize_to_loudness(sessions, float(album_loudness_target), need_no_limiter,
                                                      need_no_limiter_normalized)
        else:
            outs = [s.finalize(need_default, need_no_limiter, need_no_limiter_normalized) for s in sessions]
        if debug_enabled():
            st = sessions[0].read_state()
            debug(f"The album's {st.target_loud_pieces} loud pieces of {sum(int(s.layout.target_divisions) for s in sessions)}"
                  f" give one RMS coefficient: {to_db(st.rms_coefficient)}")
            for step in range(st.steps_done):
                debug(f"Album RMS correction #{step + 1}: {to_db(st.correction[step])}")
            if report is not None:
                from .loudness import LoudnessTarget, debug_target
                raw = report.cpu().numpy().tobytes()
                debug_target(LoudnessTarget.from_report(float(album_loudness_target),
                                                        _native.LoudnessTargetReport.from_buffer_copy(raw)))
    return outs


def main_versions(targets, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
                  need_no_limiter_normalized: bool = False):
    """Master a mix (targets[0]) and its versions -- instrumental, a cappella, TV mix, clean edit -- as linked versions
    (DESIGN.md section 4 "Linked versions"): the level and spectrum match is the main's alone, every version goes through
    the main's FIR and correction gain, and one limiter gain envelope, computed from the loudest of all their detectors
    at every frame, limits every one of them.  So main - instrumental is the vocal through the same chain.  targets:
    (N, 2) stereo arrays of ONE frame count at config.internal_sample_rate, numpy or torch; reference: samples or a
    ReferenceProfile.  Returns one (result, result_no_limiter, result_no_limiter_normalized) per target, None where not
    requested, in each target's array type.  Where no version is louder than the main at any frame, the main's outputs
    are `main`'s bit for bit.  Config(loudness_target=T) searches the main's limited output to T and gives every
    version the same drive."""
    outs = main_versions_device(targets, reference, config, need_default, need_no_limiter, need_no_limiter_normalized)
    return [tuple(None if t is None else to_host_like(t, target) for t in entry) for entry, target in zip(outs, targets)]


def versions_check(targets, config: Config) -> None:
    """The version requests main_versions refuses before any device work."""
    if len(targets) < 1:
        raise ValueError("linked versions need the main mix")
    if len(targets) - 1 > _native.MGB_MAX_VERSIONS:
        raise ValueError(f"{len(targets) - 1} versions: at most {_native.MGB_MAX_VERSIONS} are linked to one main mix")
    for target in targets:
        if target.ndim != 2 or target.shape[1] != 2:
            raise ValueError("every target must be a (frames, 2) stereo array")
    n = int(targets[0].shape[0])
    if not n > config.fft_size:
        raise ValueError(f"the main mix must be longer than fft_size ({config.fft_size} frames)")
    for k, target in enumerate(targets[1:], 1):
        if int(target.shape[0]) != n:
            raise ValueError(f"version {k} has {int(target.shape[0])} frames, the main mix {n}: linked versions share "
                             "the main's frame count")


def main_versions_device(targets, reference, config: Config, need_default: bool = True, need_no_limiter: bool = False,
                         need_no_limiter_normalized: bool = False):
    """`main_versions` with the results left on the device as float32 CUDA tensors."""
    targets = list(targets)
    versions_check(targets, config)
    profiled = isinstance(reference, ReferenceProfile)
    if profiled:
        reference.check_config(config)
    elif reference.ndim != 2 or reference.shape[1] != 2:
        raise ValueError("the reference must be a (frames, 2) stereo array")
    plan = get_plan(config)
    device = plan.device
    with torch.cuda.device(device):
        d_targets = [to_device_f32(t, device) for t in targets]
        n = int(d_targets[0].shape[0])
        if profiled:
            d_profile = reference.checked_blob(plan)
            main = TrackSession(plan, n, None)
        else:
            d_reference = to_device_f32(reference, device)
            main = TrackSession(plan, n, int(d_reference.shape[0]))
        versions = [TrackSession(plan, n, None) for _ in d_targets[1:]]

        debug_line()
        info(Code.INFO_MATCHING_LEVELS)
        debug(f"The main mix and {len(versions)} linked versions of {n} frames")
        if profiled:
            main.match_levels_profiled(d_targets[0], d_profile)
        else:
            main.match_levels(d_targets[0], d_reference)
        debug_line()
        info(Code.INFO_MATCHING_FREQS)
        main.match_frequencies(d_targets[0])
        debug_line()
        info(Code.INFO_CORRECTING_LEVELS)
        main.correct_levels()
        if versions:
            versions_match(main, versions, d_targets[1:])

        debug_line()
        info(Code.INFO_FINALIZING)
        outs, report = versions_finalize(main, [main.result] + [v.result for v in versions], need_default, need_no_limiter,
                                         need_no_limiter_normalized, config.loudness_target)
        if debug_enabled():
            _debug_scalars(main.read_state(), main.layout, reference if profiled else None)
            if report is not None:
                from .loudness import LoudnessTarget, debug_target
                raw = report.cpu().numpy().tobytes()
                debug_target(LoudnessTarget.from_report(config.loudness_target,
                                                        _native.LoudnessTargetReport.from_buffer_copy(raw)))
    return [tuple(entry) for entry in outs]
