"""Dithered PCM results on the H100: the C2 job through mg.process to 16-bit WAV (both kinds, previews included) and the
C3 job to shaped 24-bit, byte for byte against the float64 definition applied to the device's float32 output; repeats
and seeds; the batch pipeline's dithered submit_pcm; every kernel instance launched."""
import ctypes as C

import numpy as np
import pytest

import dither_oracle as do
import port

pytestmark = pytest.mark.gpu
C2_FRAMES = 44100 * 180


def wav_data(path):
    """The raw PCM of a 16/24-bit WAV: int16 (frames, 2) or uint8 (frames, 6)."""
    from matchering_b200 import wavio
    samples, _, _, _ = wavio.read_pcm(path)
    return np.array(samples)


def float_wav(path):
    from matchering_b200 import wavio
    x, _ = wavio.read(path)
    return x.astype(np.float32)  # (a FLOAT file holds the float32 output exactly)


def launches(fn):
    from matchering_b200 import _native
    lib = _native.load()
    lib.mgb_profile_enable(1)
    try:
        fn()
    finally:
        cap = 4096
        names = C.create_string_buffer(1 << 17)
        ms = (C.c_float * cap)()
        got = lib.mgb_profile_collect(names, len(names), ms, cap)
        lib.mgb_profile_enable(0)
    return names.value.decode().split("\n")[:got]


def test_c2_job_through_process_to_dithered_16_bit(tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    from matchering_b200.dither import shaping_filter
    from matchering_b200.preview_creator import preview_pieces
    t, r = port.synth_target(C2_FRAMES, 0), port.synth_reference(C2_FRAMES - 44100 * 7, 1)
    tp, rp = str(tmp_path / "t.wav"), str(tmp_path / "r.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_16")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_16")
    out = {k: str(tmp_path / f"{k}.wav") for k in ("tpdf", "shaped", "float", "plain", "pt", "pr")}
    cfg = mg.Config()
    mg.process(tp, rp, [mg.pcm16(out["tpdf"], dither="tpdf", dither_seed=1),
                        mg.pcm16(out["shaped"], dither="shaped", dither_seed=2),
                        mg.Result(out["float"], "FLOAT"), mg.pcm16(out["plain"])], config=cfg,
               preview_target=mg.pcm16(out["pt"], dither="tpdf", dither_seed=4),
               preview_result=mg.pcm16(out["pr"], dither="shaped", dither_seed=5))
    x = float_wav(out["float"])
    h = shaping_filter(44100)
    assert np.array_equal(wav_data(out["tpdf"]), do.encode(x, 16, (), 1))
    assert np.array_equal(wav_data(out["shaped"]), do.encode(x, 16, h, 2))
    assert np.array_equal(wav_data(out["plain"]), do.plain(x, 32767.0).astype(np.int16))  # undithered: as before
    # the previews: each follows its own Result
    target_in = (wav_data(tp).astype(np.float64) / 32768.0).astype(np.float32)
    _, piece_t, piece_r = preview_pieces(target_in, x, cfg)
    assert np.array_equal(wav_data(out["pt"]), do.encode(piece_t.cpu().numpy(), 16, (), 4))
    assert np.array_equal(wav_data(out["pr"]), do.encode(piece_r.cpu().numpy(), 16, h, 5))


def test_repeats_and_seeds(tmp_path):
    """The dithered file is a function of the float32 limited output and the seed: every run's file is the definition
    applied to that run's output (which may differ from run to run in the last bit, through the order of stage 3's
    float64 atomics), the encoder repeated on one output gives the same bytes, and another seed other bytes."""
    import torch

    import matchering_b200 as mg
    from matchering_b200 import dither, wavio
    from matchering_b200.engine import encode_pcm
    t, r = port.synth_target(44100 * 20, 5), port.synth_reference(44100 * 15, 6)
    tp, rp = str(tmp_path / "t.wav"), str(tmp_path / "r.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_24")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_24")
    h = dither.shaping_filter(44100)
    files, floats = [], []
    for k, seed in enumerate((7, 7, 8)):
        o, f = str(tmp_path / f"o{k}.wav"), str(tmp_path / f"f{k}.wav")
        mg.process(tp, rp, [mg.pcm16(o, dither="shaped", dither_seed=seed), mg.Result(f, "FLOAT")])
        files.append(wav_data(o))
        floats.append(float_wav(f))
        assert np.array_equal(files[-1], do.encode(floats[-1], 16, h, seed)), k
    if np.array_equal(floats[0], floats[1]):
        assert np.array_equal(files[0], files[1])
    x = torch.from_numpy(floats[0]).cuda()
    p = dither.params("shaped", 44100, 7)
    assert np.array_equal(np.array(encode_pcm(x, 16, p)), np.array(encode_pcm(x, 16, p)))
    assert np.array_equal(np.array(encode_pcm(x, 16, p)), files[0])
    assert not np.array_equal(np.array(encode_pcm(x, 16, dither.params("shaped", 44100, 8))), files[0])


def test_c3_job_to_shaped_24_bit():
    """10 minutes at 96 kHz: the device's limited output quantised by the dithered encoder, against the definition."""
    import torch

    import matchering_b200 as mg
    from matchering_b200 import dither, stages
    from matchering_b200.engine import encode_pcm
    fs = 96000
    cfg = mg.Config(internal_sample_rate=fs)
    t, r = port.synth_target(fs * 600, 10), port.synth_reference(fs * 590, 11)
    limited = stages.main_device(t, r, cfg)[0]
    got = np.array(encode_pcm(limited, 24, dither.params("shaped", fs, 2 ** 64 - 1)))
    torch.cuda.synchronize()
    x = limited.cpu().numpy()
    assert np.array_equal(got, do.encode(x, 24, dither.shaping_filter(fs), 2 ** 64 - 1))


def test_pipeline_submit_pcm_against_the_single_call_encoder():
    import torch

    import matchering_b200 as mg
    from matchering_b200 import dither
    from matchering_b200.batch import MasteringPipeline
    from matchering_b200.engine import encode_pcm
    cfg = mg.Config()
    pcm = lambda a: np.clip(np.rint(a.astype(np.float64) * 32767.0), -32768, 32767).astype(np.int16)
    pairs = [(pcm(port.synth_target(44100 * 20 - 311 * k, 40 + k)), pcm(port.synth_reference(44100 * 15, 50 + k)))
             for k in range(3)]
    max_t = max(len(t) for t, _ in pairs)
    p = dither.params("shaped", 44100, 99)
    with MasteringPipeline(cfg, max_t, 44100 * 15, depth=2, dither="shaped", dither_seed=99) as pipe:
        for t, r in pairs:
            tf = (t.astype(np.float64) / 32768.0).astype(np.float32)
            rf = (r.astype(np.float64) / 32768.0).astype(np.float32)
            o_pcm, o_f = np.empty((len(t), 2), np.int16), np.empty((len(t), 2), np.float32)
            pipe.wait(pipe.submit_pcm(t, r, o_pcm))
            pipe.wait(pipe.submit(tf, rf, o_f))
            want = np.array(encode_pcm(torch.from_numpy(o_f).cuda(), 16, p))
            assert np.array_equal(want, do.encode(o_f, 16, dither.shaping_filter(44100), 99))
            # The PCM job's float32 output is not the float32 job's to the bit on the device (stage 3's float64 atomics
            # add in any order), and a last-bit difference that moves a rounding changes the rest of its 1024-frame
            # segment.  So the two jobs' bytes must agree in all but a few segments (the emulator pins every byte).
            seg = lambda a: np.pad(a, ((0, -len(a) % 1024), (0, 0))).reshape(-1, 1024 * 2)
            differ = int(np.sum(np.any(seg(o_pcm) != seg(want), axis=1)))
            print(f"{len(t)} frames: {differ} of {len(seg(want))} segments differ")
            assert differ <= 0.01 * len(seg(want))


def test_every_instance_runs_and_matches_the_definition():
    import torch

    from matchering_b200 import _native
    from matchering_b200.engine import _stream_ptr
    lib = _native.load()
    rng = np.random.default_rng(3)
    n = 3 * 1024 * 32 + 77  # several CTAs and a partial last tile
    x = rng.uniform(-1.1, 1.1, (n, 2)).astype(np.float32)
    x[100, 0], x[200, 1], x[300, 0] = np.nan, -0.0, np.inf
    xd = torch.from_numpy(x).cuda()
    cases = []
    for bits in (16, 24):
        for taps in (0, 5, 12, 32):
            h = rng.normal(0.0, 0.4, taps)
            p = _native.DitherParams()
            p.seed, p.taps = 12345 + taps, taps
            for k, v in enumerate(h):
                p.h[k] = v
            out = torch.empty((n, 2) if bits == 16 else (n, 6), dtype=torch.int16 if bits == 16 else torch.uint8,
                              device="cuda")
            cases.append((bits, h, p, out))

    def run():
        for bits, _, p, out in cases:
            _native.check(lib, lib.mgb_pcm_encode_dithered(C.byref(p), xd.data_ptr(), n, bits, out.data_ptr(),
                                                           _stream_ptr(xd.device)))
    names = launches(run)
    for bits in (16, 24):
        for K in (0, 12, 32):
            assert f"pcm_dither_encode_kernel<{bits},{K}>" in names, (bits, K, names)
    for bits, h, p, out in cases:
        assert np.array_equal(out.cpu().numpy(), do.encode(x, bits, h, p.seed)), (bits, len(h))
