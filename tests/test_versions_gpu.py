"""Linked versions on the H100 at C2 size (3 minutes at 44.1 kHz): the main mix is seeded instrumental + vocal-like
material and three versions (instrumental, a cappella, TV mix) go with it, against the float64 restatement
(tests/versions_oracle.py), against the single job, repeated, and through mg.process_versions to WAV files."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import port  # noqa: E402
import versions_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
N = 44100 * 180


@pytest.fixture(scope="module")
def material():
    a = port.synth_target(N, 180).astype(np.float64) * 0.6
    b = port.synth_tonal(N, 181).astype(np.float64) * 0.35
    a, b = a.astype(np.float32), b.astype(np.float32)
    r = port.synth_reference(44100 * 150 + 77, 182)
    return a, b, r


def _versions(a, b):
    return [a + b, a, b, a + 0.5 * b]


@pytest.mark.parametrize("tp", [False, True], ids=["sample", "true-peak"])
def test_versions_match_the_restatement(material, tp):
    import matchering_b200 as mg
    from matchering_b200 import stages
    a, b, r = material
    cfg = mg.Config(true_peak=tp)
    targets = _versions(a, b)
    got = stages.main_versions(targets, r, cfg, True, True, True)
    tr = {}
    want = versions_oracle.main_versions(targets, r, cfg, True, True, True, trace=tr)
    for k, (g, w) in enumerate(zip(got, want)):
        for j in range(3):
            assert float(np.abs(g[j].astype(np.float64) - w[j]).max()) < TOL, (k, j)
    e = versions_oracle.envelope(tr["D"], cfg)
    vocal = versions_oracle.chain(b, tr) * e[:, None] * tr["final_coef"]
    assert float(np.abs((got[0][0].astype(np.float64) - got[1][0]) - vocal).max()) < TOL


def test_versions_at_a_loudness_target_match_the_restatement(material):
    import matchering_b200 as mg
    from matchering_b200 import stages
    a, b, r = material
    cfg = mg.Config(true_peak=True, loudness_target=-14.0)
    targets = _versions(a, b)
    got = stages.main_versions(targets, r, cfg, True, False, False)
    want = versions_oracle.main_versions(targets, r, cfg, True, False, False, loudness_target=-14.0)
    for k, (g, w) in enumerate(zip(got, want)):
        assert float(np.abs(g[0].astype(np.float64) - w[0]).max()) < TOL, k


def test_main_is_the_single_job_where_versions_are_quieter_and_repeats_are_identical(material):
    import torch
    import matchering_b200 as mg
    from matchering_b200 import stages
    a, b, r = material
    cfg = mg.Config()
    x = torch.from_numpy(a + b).cuda()
    quieter = [0.5 * x, 0.7 * x, torch.zeros_like(x)]
    got = stages.main_versions_device([x] + quieter, r, cfg, True, True, True)
    want = stages.main_device(x, r, cfg, True, True, True)
    # (stage 3's float64 atomic sums make two device runs of one job differ in the last bits: see the profile tests)
    for g, w in zip(got[0], want):
        assert float((g.double() - w.double()).abs().max()) < 1e-6
    again = stages.main_versions_device([x] + quieter, r, cfg, True, True, True)
    for e1, e2 in zip(got, again):
        for g1, g2 in zip(e1, e2):
            assert float((g1.double() - g2.double()).abs().max()) < 1e-6
    for j in range(3):
        assert torch.equal(got[1][j], 0.5 * got[0][j])
        assert not bool(got[3][j].any())


def test_process_versions_writes_files_that_null(material, tmp_path):
    from scipy.io import wavfile
    import matchering_b200 as mg
    from matchering_b200 import _native
    a, b, r = material
    n = 44100 * 30  # (a shorter job: the files' null, not the DSP, is checked here)
    paths = []
    for name, x in (("main", a[:n] + b[:n]), ("instrumental", a[:n])):
        p = str(tmp_path / f"{name}.wav")
        wavfile.write(p, 44100, x)
        paths.append(p)
    ref = str(tmp_path / "ref.wav")
    wavfile.write(ref, 44100, r)
    out24 = [str(tmp_path / f"o{k}_24.wav") for k in range(2)]
    out16 = [str(tmp_path / f"o{k}_16.wav") for k in range(2)]
    mg.process_versions(paths, ref, [[mg.pcm24(out24[k]), mg.Result(out16[k], "PCM_16", dither="shaped")]
                                     for k in range(2)])
    decode = lambda p, full: wavfile.read(p)[1].astype(np.float64) / full
    m24, i24 = (decode(p, 2.0 ** 31) for p in out24)
    m16, i16 = (decode(p, 2.0 ** 15) for p in out16)
    # the files' null: main - instrumental against the vocal through the chain, within the formats' quantisation
    from matchering_b200 import stages
    got = stages.main_versions([a[:n] + b[:n], a[:n]], r, mg.Config(), True, False, False)
    vocal = got[0][0].astype(np.float64) - got[1][0]
    assert float(np.abs((m24 - i24) - vocal).max()) < 4 * 2.0 ** -23
    assert float(np.sqrt(np.mean(((m16 - i16) - vocal) ** 2))) < 4 * 2.0 ** -15
    assert _native.MGB_MAX_VERSIONS == 8


def test_every_new_kernel_is_launched(material):
    import ctypes as C
    import matchering_b200 as mg
    from matchering_b200 import _native, stages
    a, b, r = material
    lib = _native.load()
    n = 44100 * 20
    targets = [a[:n] + b[:n], a[:n]]
    names = set()
    lib.mgb_profile_enable(1)
    try:
        for cfg in (mg.Config(), mg.Config(true_peak=True), mg.Config(limiter=mg.LimiterConfig(attack=50, hold_filter_order=2, release_filter_order=2)),
                    mg.Config(loudness_target=-14.0)):
            stages.main_versions(targets, r, cfg, True, True, True)
    finally:
        buf = C.create_string_buffer(1 << 20)
        ms = (C.c_float * 100000)()
        count = lib.mgb_profile_collect(buf, len(buf), ms, 100000)
        lib.mgb_profile_enable(0)
    names = set(buf.value.decode().split("\n"))
    assert count > 0
    for kernel in ("versions_detect_kernel", "true_peak_accumulate_kernel", "limiter_versions_kernel",
                   "limiter_wide_apply_versions_kernel"):
        assert kernel in names, kernel
