"""No kernel reads workspace, track state or output memory that it did not write in the same job.

The other end-to-end tests run every job in fresh, zero-filled buffers.  Production does not: TrackSession takes its
workspace from torch.empty (the caching allocator hands back a previous tensor's bytes), and a batch pipeline
(mgb_pipeline_*) gives each slot one workspace, one mgb_track_state and one set of staging buffers, sized for the
longest track and reused by every later one with the region offsets of that track's own layout.  Only the range
mgb_match_levels clears and the limiter words mgb_finalize clears may be read before they are written; a stale
loud-list count, conv_precise word or look-back word reads as zero in a fresh buffer and goes unnoticed there.

1. Poisoned buffers, per entry point.  Each job runs once in zero-filled buffers and once after every byte of its
   workspace, track state and outputs was written with 0xFF (NaN as a float or double, -1 as an integer), 0x7F
   (3.4e38, a huge positive integer) or seeded random bytes.  The emulator is deterministic: outputs and state must
   be bit-identical.  On the device float64 atomics may reorder the last bits of the per-piece sums: the outputs
   must be finite, within the oracle bounds and within 1e-6 (of max(1, peak)) of the clean run, the integer state
   fields equal.  The material reaches every branch that owns a workspace region: broadband (float32 convolution),
   band-limited against a bright reference (float64 convolution), gain crossing 1/kLoudMid between correction steps
   and overflowing loud lists (the correction's fall-backs to the result), a quiet reference (the limiter's
   early-out) and a mono target; every kernel launch_convolve_t can pick.

2. Mixed batches.  A scripted sequence of tracks goes through the slots of one pipeline, created with the test switch
   "poison_alloc" so that its buffers start as 0xFF.  Consecutive tracks on one slot alternate between the longest
   track, the shortest legal one and an odd length in between; references longer and shorter than the target and of
   exactly the pipeline's maximum; the float32 and float64 convolutions; limiter engaged and not; overflowing lists
   and none.  One later, shorter track has more analysis items (divisions x slots) than the track before it on its
   slot, which the pipeline's workspace sizing must allow for (pipeline.cu).  Every output is checked against the
   oracle and every returned state against the same track run alone; the same script also runs through the PCM
   entry with 16- and 24-bit widths mixed and, on the device, through batch.master_many."""
import ctypes as C

import numpy as np
import pytest

import port
from test_coloured_material import bright, brick_wall
from test_stage_parity import BY_NAME as STAGE_VARIANTS
from test_stage_parity import LOUD_MID, Variant, max_piece_seconds, regions, restore_options, set_options, spiky

TOL = 1e-5            # the suite's bound on the outputs (test_emul_kernels.py, test_gpu_parity.py)
REPEAT_TOL = 1e-6     # between two runs of one job on the device (test_pipeline_is_reproducible_and_does_not_touch_inputs)
POISONS = ["ff", "7f", "random"]
INT_FIELDS = ["steps_done", "limiter_engaged", "conv_precise", "target_loud_pieces", "reference_loud_pieces"]


# ---- poison ----------------------------------------------------------------------------------------------------
def poison_bytes(n, pattern, seed=0):
    """n bytes of a poison pattern; pattern None = zeros (the clean run)."""
    if pattern is None:
        return np.zeros(n, np.uint8)
    if pattern == "ff":
        return np.full(n, 0xFF, np.uint8)
    if pattern == "7f":
        return np.full(n, 0x7F, np.uint8)
    assert pattern == "random", pattern
    return np.random.default_rng(1234 + seed).integers(0, 256, n, dtype=np.uint8)


def ebuf(shape, dtype, pattern, seed=0):
    """An emulator buffer (256-byte aligned host memory) whose every byte holds the pattern."""
    from emul_harness import aligned
    a = aligned(shape, dtype)
    a.reshape(-1).view(np.uint8)[...] = poison_bytes(a.nbytes, pattern, seed)
    return a


def dbuf(shape, dtype, pattern, seed=0):
    """A device buffer from PyTorch's caching allocator whose every byte holds the pattern."""
    import torch
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    raw.copy_(torch.from_numpy(poison_bytes(nbytes, pattern, seed)))
    tdt = {np.float32: torch.float32, np.float64: torch.float64, np.int32: torch.int32, np.uint8: torch.uint8}[dtype]
    return raw.view(tdt).view(*shape)


def state_of(raw):
    from matchering_b200 import _native
    return _native.TrackState.from_buffer_copy(bytes(raw))


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def cuda_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def device_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from matchering_b200 import _native
    return _native.load()


# ---- material ----------------------------------------------------------------------------------------------------
# name -> (target, reference) float32 for a target of n frames and a reference of m frames
def _mono(n, m):
    t = port.synth_target(n, 13)
    t[:, 1] = t[:, 0]
    return t, port.synth_reference(m, 14)


MATERIALS = {
    "broadband": lambda n, m: (port.synth_target(n, 1), port.synth_reference(m, 2)),
    # band-limited target, bright reference: a FIR gain of ~10^3 in the empty band (test_coloured_material.py)
    "coloured": lambda n, m: (brick_wall(port.synth_target(n, 1), 2000).astype(np.float32), bright(m, 2).astype(np.float32)),
    # quiet noise with rare spikes: the correction gain crosses 1 / kLoudMid between steps (test_stage_parity.py)
    "gain_crossing": lambda n, m: (spiky(n, 5), port.synth_reference(m, 32)),
    # twice-compressed pink noise at the reference's level: more than a quarter of the mid samples reach kLoudMid
    # (edge_track's piece 1 in test_stage_parity.py)
    "overflow": lambda n, m: (np.tanh(3.0 * port.synth_reference(n, 11)), np.tanh(3.0 * port.synth_reference(m, 12))),
    # the quiet reference of tests/golden/pipeline_quiet_reference.npz: normalised, and the limiter takes its early-out
    "quiet": lambda n, m: (port.synth_target(n, 21, kind="white"),
                           (0.05 * port.synth_reference(m, 22, kind="quiet")).astype(np.float32)),
    "mono": _mono,
}
KERNELS = ["f1024_generic", "f4096_default", "f4096_ovs2", "f8192_fused", "f16384_global"]
# the limiter's chunks handed out by its atomic ticket (option "limiter_ticket") instead of the block index: the
# ticket is a workspace word that mgb_finalize clears before every limiter launch
BY_NAME = dict(STAGE_VARIANTS, f1024_limiter_ticket=Variant("f1024_limiter_ticket", 1024, {"limiter_ticket": 1},
                                                            "convolve_kernel<1024>", 2, 5))
# the other kernels and switches launch_convolve_t chooses between, with their own scratch and copy paths
OTHER_KERNELS = ["f4096_not_persistent", "f4096_no_tma", "f4096_generic", "f8192_generic", "f8192_no_tma"]


def case_geometry(material, kernel):
    """(target frames, reference frames, pieces) of one material on one kernel: pieces of at least 3F samples where
    the 4F-frame kernel exists (its choice needs them), four pieces for the gain crossing (as in test_stage_parity)."""
    F = BY_NAME[kernel].F
    if material == "gain_crossing":
        n = 16 * 3 * F + 1 if F >= 2048 else 40001
        return n, n - 5000, 4
    n, pieces = {1024: (24001, 3), 4096: (26001, 2), 8192: (18001, 2), 16384: (20001, 1)}[F]
    return n, n - n // 20, pieces


# emulator: every material on the default-size generic kernel, one material on each of the slower ones
EMULATED = [(m, "f1024_generic") for m in MATERIALS] + [
    ("broadband", "f4096_default"), ("mono", "f4096_ovs2"), ("overflow", "f8192_fused"), ("coloured", "f16384_global"),
    ("broadband", "f1024_limiter_ticket")]
# device: every material on every size, the overflowing one (float32 convolution on every kernel) on the other
# kernel choices, and two materials with the limiter's ticket
DEVICE = ([(m, k) for k in KERNELS for m in MATERIALS] + [("overflow", k) for k in OTHER_KERNELS] +
          [("broadband", "f1024_limiter_ticket"), ("overflow", "f1024_limiter_ticket")])


def limiter_words(ws_bytes, lib, plan_struct, L):
    """The limiter's tickets and look-back words as a job's workspace holds them after mgb_finalize
    (mgb_test_workspace_regions out[14], out[15])."""
    from matchering_b200 import _native
    out = (C.c_int64 * 16)()
    _native.check(lib, lib.mgb_test_workspace_regions(C.byref(plan_struct), C.byref(L), out))
    off, size = int(out[14]), int(out[15])
    assert off > 0 and size > 0 and off + size <= L.workspace_bytes
    return bytes(ws_bytes[off:off + size])


def loud_overflow(ws_bytes, lib, plan_struct, L):
    """Per piece: did the loud list overflow (count > capacity)?  From a job's workspace after the stage calls."""
    reg = regions(lib, plan_struct, L)
    counts = np.frombuffer(ws_bytes, np.uint32, L.target_divisions, reg["loud_count"])
    return counts > reg["loud_capacity"]


def check_premise(material, st, overflow, t, F, outs=None):
    """What makes the material worth running: the branch it is there to reach was taken.  The float32 convolution
    runs for the overflowing material on every kernel and for the broadband one up to fft_size 4096 (on these short
    tracks its FIR peaks put the larger kernels' estimate above kConvPreciseError, convolve.cu)."""
    steps = st.steps_done
    gains = np.cumprod([st.correction[i] for i in range(steps)])
    if material == "coloured":
        assert st.conv_precise == 1 and st.limiter_engaged == 1
    elif material == "overflow" or (material == "broadband" and F <= 4096):
        assert st.conv_precise == 0, material
    if material == "gain_crossing":
        assert gains[0] * LOUD_MID < 1 < gains[-2] * LOUD_MID, gains
    if material == "overflow":
        assert overflow.any(), overflow
    if material == "quiet":
        assert st.limiter_engaged == 0 and st.final_amplitude_coef < 1.0
    if material != "quiet":
        assert st.limiter_engaged == 1, material
    if material == "mono":
        assert np.array_equal(t[:, 0], t[:, 1])
        if outs is not None:
            assert all(np.array_equal(o[:, 0], o[:, 1]) for o in outs)


def oracle_outputs(t, r, cfg):
    return port.main(t.astype(np.float64), r.astype(np.float64), port.config_from(cfg), True, True, True)


def check_against_oracle(outs, want):
    """Limited output within 1e-5; the unlimited ones within 1e-5 of max(1, peak) (a pre-limiter peak above 1 is
    stored in float32 with an ulp above 1e-7, test_coloured_material.py)."""
    err = float(np.abs(outs[0].astype(np.float64) - want[0]).max())
    assert err <= TOL, ("limited", err)
    worst = err
    for name, got, w in (("no_limiter", outs[1], want[1]), ("normalized", outs[2], want[2])):
        e = float(np.abs(got.astype(np.float64) - w).max()) / max(1.0, float(np.abs(w).max()))
        assert e <= TOL, (name, e)
        worst = max(worst, e)
    return worst


def check_device_repeat(clean, dirty, clean_state, dirty_state):
    """The device's clean-vs-poisoned bound: finite, within 1e-6 of max(1, peak), integer state fields equal."""
    worst = 0.0
    for a, b in zip(clean, dirty):
        assert np.isfinite(b).all()
        e = float(np.abs(a.astype(np.float64) - b).max()) / max(1.0, float(np.abs(a).max()))
        assert e <= REPEAT_TOL, e
        worst = max(worst, e)
    for f in INT_FIELDS:
        assert getattr(clean_state, f) == getattr(dirty_state, f), f
    return worst


# ---- the four stage calls on poisoned buffers --------------------------------------------------------------------
def stages_emulated(cfg, t, r, pattern):
    from emul_harness import aligned_copy, emul_lib, get_emul_plan, ptr
    from matchering_b200 import _native
    lib = emul_lib()
    ep = get_emul_plan(cfg)
    T, R = len(t), len(r)
    L = ep.layout(T, R)
    ws = ebuf((L.workspace_bytes,), np.uint8, pattern, 0)
    tgt, ref = aligned_copy(t, np.float32), aligned_copy(r, np.float32)
    result = ebuf((T, 2), np.float32, pattern, 1)
    fir = ebuf((2, cfg.fft_size), np.float64, pattern, 2)
    state = ebuf((C.sizeof(_native.TrackState),), np.uint8, pattern, 3)
    outs = [ebuf((T, 2), np.float32, pattern, 4 + k) for k in range(3)]
    P, LL, S = C.byref(ep.struct), C.byref(L), ptr(state)
    _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), S, None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(result), ptr(fir), ptr(ws), S, None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), S, None))
    _native.check(lib, lib.mgb_finalize(P, LL, ptr(result), *(ptr(o) for o in outs), ptr(ws), S, None))
    return dict(outs=[np.array(o) for o in outs], state=state.tobytes(), result=np.array(result), fir=np.array(fir),
                overflow=loud_overflow(ws.tobytes(), lib, ep.struct, L), limiter=limiter_words(ws.tobytes(), lib, ep.struct, L),
                L=L)


def stages_device(cfg, t, r, pattern):
    import torch
    from matchering_b200 import _native
    from matchering_b200.engine import get_plan
    plan = get_plan(cfg)
    lib = plan.lib
    T, R = len(t), len(r)
    L = plan.layout(T, R)
    ws = dbuf((L.workspace_bytes,), np.uint8, pattern, 0)
    tgt, ref = torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda()
    result = dbuf((T, 2), np.float32, pattern, 1)
    fir = dbuf((2, cfg.fft_size), np.float64, pattern, 2)
    state = dbuf((C.sizeof(_native.TrackState),), np.uint8, pattern, 3)
    outs = [dbuf((T, 2), np.float32, pattern, 4 + k) for k in range(3)]
    P, LL, S, st = C.byref(plan.struct), C.byref(L), state.data_ptr(), cuda_stream()
    _native.check(lib, lib.mgb_match_levels(P, LL, tgt.data_ptr(), ref.data_ptr(), ws.data_ptr(), S, st))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, tgt.data_ptr(), result.data_ptr(), fir.data_ptr(), ws.data_ptr(),
                                                 S, st))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ws.data_ptr(), S, st))
    _native.check(lib, lib.mgb_finalize(P, LL, result.data_ptr(), *(o.data_ptr() for o in outs), ws.data_ptr(), S, st))
    torch.cuda.synchronize()
    wb = ws.cpu().numpy().tobytes()
    return dict(outs=[o.cpu().numpy() for o in outs], state=state.cpu().numpy().tobytes(), result=result.cpu().numpy(),
                fir=fir.cpu().numpy(), overflow=loud_overflow(wb, lib, plan.struct, L), limiter=limiter_words(wb, lib, plan.struct, L),
                L=L)


def case_config(material, kernel, device):
    import matchering_b200 as mg
    F = BY_NAME[kernel].F
    n, m, pieces = case_geometry(material, kernel)
    kw = dict(fft_size=F, max_piece_size=max_piece_seconds(n, pieces))
    return (mg.Config(**kw) if device else port.OracleConfig(**kw)), n, m


_CLEAN = {}


def stage_case(material, kernel, device, pattern):
    """(clean run, poisoned run, t, r, cfg) of one material on one kernel; the clean run and the oracle are kept."""
    variant = BY_NAME[kernel]
    cfg, n, m = case_config(material, kernel, device)
    t, r = MATERIALS[material](n, m)
    run = stages_device if device else stages_emulated
    if device:
        lib = device_lib()
    else:
        from emul_harness import emul_lib
        lib = emul_lib()
    set_options(lib, variant.options)
    try:
        key = (material, kernel, device)
        if key not in _CLEAN:
            clean = run(cfg, t, r, None)
            assert variant.expected_ovs(clean["L"].target_piece) == variant.ovs
            st = state_of(clean["state"])
            check_premise(material, st, clean["overflow"], t, variant.F, outs=clean["outs"])
            clean["err"] = check_against_oracle(clean["outs"], oracle_outputs(t, r, cfg))
            _CLEAN[key] = clean
        dirty = run(cfg, t, r, pattern)
    finally:
        restore_options(lib)
        lib.mgb_set_option(b"limiter_ticket", 0)
    return _CLEAN[key], dirty, t, r, cfg


@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("material,kernel", EMULATED)
def test_stage_calls_on_poisoned_buffers_emulated(material, kernel, pattern):
    clean, dirty, _, _, _ = stage_case(material, kernel, False, pattern)
    for k, (a, b) in enumerate(zip(clean["outs"], dirty["outs"])):
        assert same_bits(a, b), ("output", k)
    assert same_bits(clean["result"], dirty["result"]) and same_bits(clean["fir"], dirty["fir"])
    assert clean["state"] == dirty["state"], (state_of(clean["state"]), state_of(dirty["state"]))
    # what the limiter leaves in its tickets and look-back words: mgb_finalize cleared them before its launch
    assert clean["limiter"] == dirty["limiter"]


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("material,kernel", DEVICE)
def test_stage_calls_on_poisoned_buffers_device(material, kernel, pattern):
    clean, dirty, t, r, cfg = stage_case(material, kernel, True, pattern)
    check_against_oracle(dirty["outs"], oracle_outputs(t, r, cfg))
    worst = check_device_repeat(clean["outs"] + [clean["result"]], dirty["outs"] + [dirty["result"]],
                                state_of(clean["state"]), state_of(dirty["state"]))
    # the limiter's chunk ticket counted from the zero mgb_finalize wrote (the look-back words' flags depend on
    # the order the chunks ran in, on the device)
    ticket = np.frombuffer(dirty["limiter"], np.int32, 1)[0]
    assert ticket == np.frombuffer(clean["limiter"], np.int32, 1)[0]
    assert (ticket > 0) == ("limiter_ticket" in BY_NAME[kernel].options), ticket
    print(f"{material} {kernel} {pattern}: clean vs poisoned {worst:.2e}, clean vs oracle {clean['err']:.2e}")


# ---- the single-call host entries --------------------------------------------------------------------------------
HOST_CASES = ["broadband", "quiet"]


def host_case(material):
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=max_piece_seconds(24001, 3))
    t, r = MATERIALS[material](24001, 21601)
    return cfg, t, r


def process_host_emulated(cfg, t, r, pattern):
    from emul_harness import emul_lib, get_emul_plan, ptr
    from matchering_b200 import _native
    lib = emul_lib()
    ep = get_emul_plan(cfg)
    T, R = len(t), len(r)
    L = ep.layout(T, R)
    d = dict(t=ebuf((T, 2), np.float32, pattern, 0), r=ebuf((R, 2), np.float32, pattern, 1),
             res=ebuf((T, 2), np.float32, pattern, 2), out=ebuf((T, 2), np.float32, pattern, 3),
             ws=ebuf((L.workspace_bytes,), np.uint8, pattern, 4), st=ebuf((C.sizeof(_native.TrackState),), np.uint8, pattern, 5))
    outs = [np.frombuffer(poison_bytes(T * 8, pattern, 6 + k).tobytes(), np.float32).reshape(T, 2).copy() for k in range(3)]
    state = _native.TrackState.from_buffer_copy(poison_bytes(C.sizeof(_native.TrackState), pattern, 9).tobytes())
    _native.check(lib, lib.mgb_process_host(C.byref(ep.struct), C.byref(L), t.ctypes.data, r.ctypes.data, *(o.ctypes.data for o in outs),
                                            ptr(d["t"]), ptr(d["r"]), ptr(d["res"]), ptr(d["out"]), ptr(d["ws"]), ptr(d["st"]),
                                            C.byref(state), None))
    return outs, bytes(state)


def process_host_device(cfg, t, r, pattern):
    import torch
    from matchering_b200 import _native
    from matchering_b200.engine import get_plan
    plan = get_plan(cfg)
    lib = plan.lib
    T, R = len(t), len(r)
    L = plan.layout(T, R)
    d = dict(t=dbuf((T, 2), np.float32, pattern, 0), r=dbuf((R, 2), np.float32, pattern, 1),
             res=dbuf((T, 2), np.float32, pattern, 2), out=dbuf((T, 2), np.float32, pattern, 3),
             ws=dbuf((L.workspace_bytes,), np.uint8, pattern, 4), st=dbuf((C.sizeof(_native.TrackState),), np.uint8, pattern, 5))
    outs = [np.frombuffer(poison_bytes(T * 8, pattern, 6 + k).tobytes(), np.float32).reshape(T, 2).copy() for k in range(3)]
    state = _native.TrackState.from_buffer_copy(poison_bytes(C.sizeof(_native.TrackState), pattern, 9).tobytes())
    _native.check(lib, lib.mgb_process_host(C.byref(plan.struct), C.byref(L), t.ctypes.data, r.ctypes.data,
                                            *(o.ctypes.data for o in outs), *(d[k].data_ptr() for k in ("t", "r", "res", "out", "ws", "st")),
                                            C.byref(state), cuda_stream()))
    torch.cuda.synchronize()
    return outs, bytes(state)


def stages_main_host_run(lib, io, plan_struct, L, t, r, bufs, pattern, stream):
    """mgb_stages_main_host with float64 host arrays in and out (the reference's seam)."""
    from matchering_b200 import _native
    T = len(t)
    ht, hr = t.astype(np.float64), r.astype(np.float64)
    outs = [np.frombuffer(poison_bytes(T * 16, pattern, 10 + k).tobytes(), np.float64).reshape(T, 2).copy() for k in range(3)]
    state = _native.TrackState.from_buffer_copy(poison_bytes(C.sizeof(_native.TrackState), pattern, 13).tobytes())
    _native.check(lib, lib.mgb_stages_main_host(io, C.byref(plan_struct), C.byref(L), ht.ctypes.data, hr.ctypes.data, 8,
                                                *(o.ctypes.data for o in outs), 8, C.byref(bufs), C.byref(state), stream))
    return outs, bytes(state)


def host_buffers(alloc, T, R, ws_bytes, pattern):
    from matchering_b200 import _native
    keep = dict(t=alloc((T, 2), np.float32, pattern, 20), r=alloc((R, 2), np.float32, pattern, 21),
                res=alloc((T, 2), np.float32, pattern, 22), out=alloc((T, 2), np.float32, pattern, 23),
                wide=alloc((T, 2), np.float64, pattern, 24), ws=alloc((ws_bytes,), np.uint8, pattern, 25),
                st=alloc((C.sizeof(_native.TrackState),), np.uint8, pattern, 26))
    addr = {k: (v.ctypes.data if isinstance(v, np.ndarray) else v.data_ptr()) for k, v in keep.items()}
    b = _native.HostBuffers()
    b.d_target_lr, b.d_reference_lr, b.d_result_lr, b.d_out_lr = addr["t"], addr["r"], addr["res"], addr["out"]
    b.d_wide, b.d_workspace, b.d_state = addr["wide"], addr["ws"], addr["st"]
    return b, keep


@pytest.fixture(scope="module")
def emul_io():
    from emul_harness import emul_lib
    from matchering_b200 import _native
    lib = emul_lib()
    h = C.c_void_p()
    _native.check(lib, lib.mgb_host_io_create(3, 4096, 3, C.byref(h)))
    yield h
    lib.mgb_host_io_destroy(h)


@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("material", HOST_CASES)
def test_host_entries_on_poisoned_buffers_emulated(material, pattern, emul_io):
    """mgb_process_host and mgb_stages_main_host: every device staging buffer, the state and the host outputs."""
    from emul_harness import emul_lib, get_emul_plan
    cfg, t, r = host_case(material)
    want = oracle_outputs(t, r, cfg)
    lib = emul_lib()
    L = get_emul_plan(cfg).layout(len(t), len(r))
    def run(p):
        outs, st = process_host_emulated(cfg, t, r, p)
        bufs, keep = host_buffers(ebuf, len(t), len(r), L.workspace_bytes, p)
        outs64, st64 = stages_main_host_run(lib, emul_io, get_emul_plan(cfg).struct, L, t, r, bufs, p, None)
        return outs, st, outs64, st64
    key = ("host", material)
    if key not in _CLEAN:
        _CLEAN[key] = run(None)
    (o0, s0, w0, t0), (o1, s1, w1, t1) = _CLEAN[key], run(pattern)
    check_premise(material, state_of(s0), np.zeros(1, bool), t, cfg.fft_size)
    check_against_oracle(o0, want)
    assert all(same_bits(a, b) for a, b in zip(o0, o1)) and s0 == s1
    assert all(same_bits(a, b) for a, b in zip(w0, w1)) and t0 == t1
    assert all(same_bits(a.astype(np.float64), b) for a, b in zip(o0, w0))  # both entries: the same job


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("material", HOST_CASES)
def test_host_entries_on_poisoned_buffers_device(material, pattern):
    import matchering_b200 as mg
    from matchering_b200.engine import HostIO, get_plan
    device_lib()
    cfg, t, r = host_case(material)
    want = oracle_outputs(t, r, cfg)
    mcfg = mg.Config(fft_size=cfg.fft_size, max_piece_size=max_piece_seconds(len(t), 3))
    plan = get_plan(mcfg)
    L = plan.layout(len(t), len(r))
    io = HostIO.get()
    runs = {}
    for p in (None, pattern):
        outs, st = process_host_device(mcfg, t, r, p)
        bufs, keep = host_buffers(dbuf, len(t), len(r), L.workspace_bytes, p)
        with io.lock:
            outs64, st64 = stages_main_host_run(plan.lib, io.handle, plan.struct, L, t, r, bufs, p, cuda_stream())
        runs[p] = (outs, state_of(st), outs64, state_of(st64))
    (o0, s0, w0, t0), (o1, s1, w1, t1) = runs[None], runs[pattern]
    check_premise(material, s0, np.zeros(1, bool), t, cfg.fft_size)
    for outs in (o0, o1, w0, w1):
        check_against_oracle(outs, want)
    worst = check_device_repeat(o0, o1, s0, s1)
    worst = max(worst, check_device_repeat(w0, w1, t0, t1))
    print(f"host entries {material} {pattern}: clean vs poisoned {worst:.2e}")


# ---- the standalone limiter --------------------------------------------------------------------------------------
LIMIT_FRAMES = 4608 * 5 + 77  # several limiter chunks: their look-back words are in the workspace


def limiter_inputs(scale):
    return (scale * port.synth_limiter_input(LIMIT_FRAMES, 5)).astype(np.float32)


def limit_calls(lib, params, x, alloc, addr, pattern, io, stream, sync):
    """mgb_limit, mgb_test_limiter_gains and mgb_limit_host on one input.  -> {entry: (output, engaged)}"""
    n = len(x)
    ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    got = {}
    for entry in ("limit", "gains"):
        xin = alloc((n, 2), np.float32, None, 0)
        xin_host = x if isinstance(xin, np.ndarray) else None
        if xin_host is not None:
            xin[...] = x
        else:
            import torch
            xin.copy_(torch.from_numpy(x))
        out, ws, flag = alloc((n, 2), np.float32, pattern, 30), alloc((ws_bytes,), np.uint8, pattern, 31), alloc((1,), np.int32, pattern, 32)
        fn = lib.mgb_limit if entry == "limit" else lib.mgb_test_limiter_gains
        from matchering_b200 import _native
        _native.check(lib, fn(C.byref(params), addr(xin), addr(out), n, addr(ws), ws_bytes, addr(flag), stream))
        sync()
        got[entry] = (np.array(out) if isinstance(out, np.ndarray) else out.cpu().numpy(),
                      int(np.array(flag)[0] if isinstance(flag, np.ndarray) else flag.cpu().numpy()[0]))
    d_in, d_out, wide = alloc((n, 2), np.float32, pattern, 33), alloc((n, 2), np.float32, pattern, 34), alloc((n, 2), np.float64, pattern, 35)
    ws, flag = alloc((ws_bytes,), np.uint8, pattern, 36), alloc((1,), np.int32, pattern, 37)
    h_in = x.astype(np.float64)
    fill = np.frombuffer(poison_bytes(n * 16, pattern, 38).tobytes(), np.float64).reshape(n, 2)
    h_out = fill.copy()
    engaged = C.c_int32(-7)
    from matchering_b200 import _native
    _native.check(lib, lib.mgb_limit_host(io, C.byref(params), h_in.ctypes.data, 8, h_out.ctypes.data, 8, n, addr(d_in), addr(d_out),
                                          addr(wide), addr(ws), ws_bytes, addr(flag), C.byref(engaged), stream))
    if engaged.value == 0:
        assert same_bits(h_out, fill)  # not written: the caller returns its input object (hyrax.py:83-85)
    got["limit_host"] = (h_out, engaged.value)
    return got


def check_limit_results(clean, dirty, x, device):
    cfg = port.OracleConfig()
    for entry in clean:
        (a, ea), (b, eb) = clean[entry], dirty[entry]
        assert ea == eb, entry
        if entry == "limit_host" and ea == 0:
            continue
        if entry != "gains":
            want = port.limit(x.astype(np.float64), cfg) if ea else x.astype(np.float64)
            assert np.abs(a - want).max() < 3e-7 and np.abs(b - want).max() < 3e-7, entry
        if device:
            assert np.isfinite(b).all() and np.abs(a.astype(np.float64) - b).max() <= REPEAT_TOL, entry
        else:
            assert same_bits(a, b), entry


@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("scale", [1.0, 0.2])
def test_limiter_entries_on_poisoned_buffers_emulated(scale, pattern, emul_io):
    from emul_harness import emul_lib, limiter_params, ptr
    from matchering_b200 import plan as plan_mod
    lib = emul_lib()
    params = limiter_params(plan_mod.limiter_constants(port.OracleConfig()))
    x = limiter_inputs(scale)
    runs = [limit_calls(lib, params, x, ebuf, ptr, p, emul_io, None, lambda: None) for p in (None, pattern)]
    assert runs[0]["limit"][1] == (1 if scale == 1.0 else 0)  # engaged, and the early-out
    check_limit_results(runs[0], runs[1], x, device=False)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", POISONS)
@pytest.mark.parametrize("scale", [1.0, 0.2])
def test_limiter_entries_on_poisoned_buffers_device(scale, pattern):
    import torch
    import matchering_b200 as mg
    from matchering_b200.engine import HostIO, get_plan
    device_lib()
    plan = get_plan(mg.Config())
    params = plan.struct.limiter
    x = limiter_inputs(scale)
    io = HostIO.get()
    runs = []
    for p in (None, pattern):
        with io.lock:
            runs.append(limit_calls(plan.lib, params, x, dbuf, lambda t: t.data_ptr(), p, io.handle, cuda_stream(),
                                    torch.cuda.synchronize))
    assert runs[0]["limit"][1] == (1 if scale == 1.0 else 0)
    check_limit_results(runs[0], runs[1], x, device=True)


# ---- the smoothing operator ----------------------------------------------------------------------------------------
def operator_struct(plan_struct):
    from matchering_b200 import _native
    s = _native.Plan.from_buffer_copy(plan_struct)
    s.d_smooth_op, s.d_smooth_op_rows = None, None
    return s


@pytest.mark.parametrize("pattern", POISONS)
def test_build_operator_on_poisoned_workspace_emulated(pattern):
    """mgb_plan_build_operator writes the same operator whatever its workspace and output held before."""
    from emul_harness import emul_lib, get_emul_plan, ptr
    from matchering_b200 import _native
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=512, lin_log_oversampling=1, lowess_frac=0.06)  # a small grid: the emulated build is slow
    s = operator_struct(get_emul_plan(cfg).struct)  # (the cached plan keeps the tables s points to alive)
    ws_bytes = int(lib.mgb_plan_operator_workspace_bytes(C.byref(s)))
    n = cfg.fft_size // 2 + 1

    def build(p):
        ws, op = ebuf((ws_bytes,), np.uint8, p, 40), ebuf((n, n), np.float64, p, 41)
        _native.check(lib, lib.mgb_plan_build_operator(C.byref(s), ptr(op), ptr(ws), ws_bytes, None))
        return np.array(op)
    if "operator" not in _CLEAN:
        _CLEAN["operator"] = build(None)
    clean = _CLEAN["operator"]
    assert np.isfinite(clean).all() and np.abs(clean).max() > 0
    assert same_bits(clean, build(pattern))


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", POISONS)
def test_build_operator_on_poisoned_workspace_device(pattern):
    import torch
    import matchering_b200 as mg
    from matchering_b200 import _native
    from matchering_b200.engine import get_plan
    lib = device_lib()
    cfg = mg.Config()
    s = operator_struct(get_plan(cfg).struct)
    ws_bytes = int(lib.mgb_plan_operator_workspace_bytes(C.byref(s)))
    n = cfg.fft_size // 2 + 1
    ops = []
    for p in (None, pattern):
        ws, op = dbuf((ws_bytes,), np.uint8, p, 40), dbuf((n, n), np.float64, p, 41)
        _native.check(lib, lib.mgb_plan_build_operator(C.byref(s), op.data_ptr(), ws.data_ptr(), ws_bytes, cuda_stream()))
        torch.cuda.synchronize()
        ops.append(op.cpu().numpy())
    assert np.isfinite(ops[1]).all() and np.abs(ops[0]).max() > 0
    assert np.abs(ops[0] - ops[1]).max() <= 1e-15 * np.abs(ops[0]).max()


# ---- mixed batches through the reused slots ------------------------------------------------------------------------
# Per slot, in submission order: (target length, reference length, material).  Lengths: "max" = the pipeline's
# max_target_frames, "short" = the shortest legal track (test_shortest_legal_tracks_single_piece), "mid" = an odd
# length between them with more analysis items than "max" on this machine.  References: "max" = max_reference_frames
# (longer than any target), "longer" / "shorter" than the track's target.  Slot k of a depth-d pipeline takes
# submissions k, k + d, k + 2d, ...
SLOT_SCRIPTS = [
    [("max", "max", "overflow"), ("short", "shorter", "quiet"), ("mid", "longer", "coloured"), ("max", "shorter", "broadband")],
    [("max", "shorter", "gain_crossing"), ("mid", "max", "broadband"), ("short", "longer", "mono"), ("max", "max", "coloured")],
    [("mid", "shorter", "coloured"), ("max", "longer", "broadband"), ("short", "max", "quiet")],
]
BATCH_F = 1024
SHORT = (1500, 1025)  # test_shortest_legal_tracks_single_piece: one piece, one analysis frame


def items(L):
    return L.target_divisions * L.target_slots


def batch_lengths(layout, piece_seconds):
    """(max, mid): the shortest odd length of d - 1/2 pieces (d = 2 .. 8) that some shorter odd length of that form
    beats in analysis items (divisions x slots), and the longest such shorter length.  Slots are 3 * SMs / divisions
    rounded down (mgb_track_layout_init), so which lengths do this depends on the SM count: the layout decides."""
    piece = piece_seconds * 44100
    cands = [int((d - 0.5) * piece) | 1 for d in range(2, 9)]
    count = {n: items(layout(n, n)) for n in cands}
    for longest in cands:
        beaten_by = [n for n in cands if n < longest and count[n] > count[longest]]
        if beaten_by:
            return longest, max(beaten_by)
    raise AssertionError(f"no shorter track with more analysis items among {count}")


def batch_script(layout, depth, piece_seconds):
    """The submissions in order: dicts of slot, lengths, material, target and reference."""
    T_MAX, T_MID = batch_lengths(layout, piece_seconds)
    R_MAX = T_MAX + 2000
    lengths = {"max": T_MAX, "short": SHORT[0], "mid": T_MID}
    per_slot = SLOT_SCRIPTS[:depth]
    subs = []
    for k in range(sum(len(s) for s in per_slot)):
        slot, turn = k % depth, k // depth
        tk, rk, material = per_slot[slot][turn]
        T = lengths[tk]
        R = {"max": R_MAX, "longer": T + 777, "shorter": SHORT[1] if tk == "short" else T - T // 8}[rk]
        t, r = MATERIALS[material](T, R)
        subs.append(dict(slot=slot, turn=turn, tkey=tk, rkey=rk, material=material, t=t, r=r))
    return subs, T_MAX, R_MAX


def check_script_premises(subs, alone, layout, T_MAX, R_MAX, depth):
    """What the script is there to reach, from each track run alone: every slot reused at least twice, and on its
    slots consecutive tracks that differ in length, reference, convolution path, limiter, lists and items."""
    per_slot = {}
    for s, a in zip(subs, alone):
        st = state_of(a["state"])
        check_premise(s["material"], st, a["overflow"], s["t"], BATCH_F)
        s.update(L=a["L"], precise=st.conv_precise, engaged=st.limiter_engaged, overflow=bool(a["overflow"].any()),
                 early_out=st.limiter_engaged == 0 and st.final_amplitude_coef < 1.0)
        per_slot.setdefault(s["slot"], []).append(s)
    assert sorted(per_slot) == list(range(depth)) and all(len(v) >= 3 for v in per_slot.values())
    assert max(len(s["t"]) for s in subs) == T_MAX and max(len(s["r"]) for s in subs) == R_MAX
    found = dict(lengths=False, refs=False, conv=False, limiter=False, overflow=False, early_out=False, items=False)
    for seq in per_slot.values():
        for a, b, c in zip(seq, seq[1:], seq[2:]):
            found["lengths"] |= [len(x["t"]) for x in (a, b, c)] == [T_MAX, SHORT[0], len(c["t"])] and len(c["t"]) % 2 == 1 \
                and SHORT[0] < len(c["t"]) < T_MAX
            kinds = {("max" if len(x["r"]) == R_MAX else "longer" if len(x["r"]) > len(x["t"]) else "shorter") for x in (a, b, c)}
            found["refs"] |= kinds == {"max", "longer", "shorter"} or (len(a["r"]) == R_MAX and len(b["r"]) < len(b["t"])
                                                                      and len(c["r"]) > len(c["t"]))
            found["conv"] |= [a["precise"], b["precise"], c["precise"]] == [0, 1, 0]
            found["limiter"] |= [a["engaged"], b["engaged"], c["engaged"]] == [1, 0, 1]
            found["early_out"] |= b["early_out"] and a["engaged"] == 1 and c["engaged"] == 1
        for a, b in zip(seq, seq[1:]):
            found["overflow"] |= a["overflow"] and not b["overflow"]
            found["items"] |= len(b["t"]) < len(a["t"]) and items(b["L"]) > items(a["L"])
    assert all(found.values()), found


def pcm_encode(x, bits):
    x = np.asarray(x, np.float64)
    if bits == 16:
        return np.clip(np.rint(x * 32767.0), -32768, 32767).astype(np.int16)
    q = np.clip(np.rint(x * 8388607.0), -8388608, 8388607).astype(np.int64) & 0xFFFFFF
    return np.stack([q & 0xFF, (q >> 8) & 0xFF, (q >> 16) & 0xFF], axis=-1).astype(np.uint8).reshape(len(x), 6)


def pcm_decode(b, bits):
    """What mgb_pcm_decode yields (libsndfile's read: x / 2^(bits-1)), in float64."""
    if bits == 16:
        return b.astype(np.float64) / 32768.0
    v = b.reshape(-1, 3).astype(np.int64)
    v = v[:, 0] | (v[:, 1] << 8) | (v[:, 2] << 16)
    v = np.where(v >= 1 << 23, v - (1 << 24), v)
    return (v / 8388608.0).reshape(-1, 2)


def pcm_widths(k):
    """(target, reference, output) bits of submission k: every combination turns up, and consecutive
    submissions on a slot differ."""
    return (16, 24)[k % 2], (24, 16)[(k // 2) % 2], (16, 24)[(k // 3) % 2]


class Pipe:
    """mgb_pipeline_* over the emulator or the device, created with poisoned slot buffers."""

    def __init__(self, lib, plan_struct, max_t, max_r, depth, stream_sync=lambda: None):
        from matchering_b200 import _native
        self.lib, self.h, self.sync = lib, C.c_void_p(), stream_sync
        _native.check(lib, lib.mgb_set_option(b"poison_alloc", 1))
        try:
            _native.check(lib, lib.mgb_pipeline_create(C.byref(plan_struct), max_t, max_r, depth, C.byref(self.h)))
        finally:
            lib.mgb_set_option(b"poison_alloc", 0)
        self.keep = {}

    def submit(self, t, r, out):
        from matchering_b200 import _native
        slot = C.c_int32(-1)
        _native.check(self.lib, self.lib.mgb_pipeline_submit(self.h, t.ctypes.data, len(t), r.ctypes.data, len(r),
                                                             out.ctypes.data, C.byref(slot)))
        self.keep[slot.value] = (t, r, out)
        return slot.value

    def submit_pcm(self, t, tb, r, rb, out, ob):
        from matchering_b200 import _native
        slot = C.c_int32(-1)
        _native.check(self.lib, self.lib.mgb_pipeline_submit_pcm(self.h, t.ctypes.data, tb, len(t), r.ctypes.data, rb, len(r),
                                                                 out.ctypes.data, ob, C.byref(slot)))
        self.keep[slot.value] = (t, r, out)
        return slot.value

    def wait(self, slot):
        from matchering_b200 import _native
        st = _native.TrackState()
        _native.check(self.lib, self.lib.mgb_pipeline_wait(self.h, slot, C.byref(st)))
        return st

    def close(self):
        self.lib.mgb_pipeline_destroy(self.h)


def run_script(pipe, subs, pcm=False):
    """Submits every track to a fresh pipeline (float32 or PCM entry), collecting a slot's previous result only when
    the slot comes round again (as a caller keeping `depth` tracks in flight does; the next submit there overwrites
    the slot's state), then destroys the pipeline.  -> (outputs, states, slots)"""
    try:
        return _run_script(pipe, subs, pcm)
    finally:
        pipe.close()


def _run_script(pipe, subs, pcm):
    outs, states, slots = [None] * len(subs), [None] * len(subs), []
    pending = {}
    for k, s in enumerate(subs):
        if s["slot"] in pending:
            states[pending.pop(s["slot"])] = pipe.wait(s["slot"])
        if pcm:
            tb, rb, ob = pcm_widths(k)
            t, r = pcm_encode(s["t"], tb), pcm_encode(s["r"], rb)
            out = np.zeros((len(t), 2), np.int16) if ob == 16 else np.zeros((len(t), 6), np.uint8)
            slot = pipe.submit_pcm(t, tb, r, rb, out, ob)
            s["pcm"] = (t, tb, r, rb, ob)
        else:
            out = np.full((len(s["t"]), 2), np.nan, np.float32)
            slot = pipe.submit(np.ascontiguousarray(s["t"]), np.ascontiguousarray(s["r"]), out)
        assert slot == s["slot"], (k, slot)
        pending[slot] = k
        outs[k] = out
        slots.append(slot)
    for slot, j in pending.items():
        states[j] = pipe.wait(slot)
    return outs, states, slots


def check_pcm_outputs(subs, outs, cfg):
    """Decode -> oracle -> compare within the float bound plus one LSB of the output (test_pipeline_pcm_entry)."""
    worst = 0.0
    for s, out in zip(subs, outs):
        t, tb, r, rb, ob = s["pcm"]
        want = port.main(pcm_decode(t, tb), pcm_decode(r, rb), port.config_from(cfg))[0]
        full = 32767.0 if ob == 16 else 8388607.0
        got = pcm_decode(out, ob) * ((full + 1) / full)
        e = float(np.abs(got - want).max())
        assert e <= TOL + 1.0 / full, (s["material"], ob, e)
        worst = max(worst, e)
    return worst


BATCH_PIECE_EMULATED = 0.25  # seconds: pieces of 10-11k samples, 8 or more analysis frames at fft_size 1024
BATCH_PIECE_DEVICE = 2.0     # pieces long enough that 3 * SMs / divisions slots fit in every one of them


def test_mixed_batch_through_reused_slots_emulated():
    from emul_harness import emul_lib, get_emul_plan
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=BATCH_F, max_piece_size=BATCH_PIECE_EMULATED)
    ep = get_emul_plan(cfg)
    depth = 2
    subs, T_MAX, R_MAX = batch_script(ep.layout, depth, BATCH_PIECE_EMULATED)
    alone = [stages_emulated(cfg, s["t"], s["r"], None) for s in subs]
    check_script_premises(subs, alone, ep.layout, T_MAX, R_MAX, depth)
    outs, states, slots = run_script(Pipe(lib, ep.struct, T_MAX, R_MAX, depth), subs)
    pcm_outs, _, pcm_slots = run_script(Pipe(lib, ep.struct, T_MAX, R_MAX, depth), subs, pcm=True)
    assert [slots.count(k) for k in range(depth)] == [len(SLOT_SCRIPTS[k]) for k in range(depth)] and pcm_slots == slots
    for s, a, out, st in zip(subs, alone, outs, states):
        assert same_bits(out, a["outs"][0]), (s["material"], s["tkey"])
        assert bytes(st) == a["state"], (s["material"], s["tkey"], st, state_of(a["state"]))
        want = port.main(s["t"].astype(np.float64), s["r"].astype(np.float64), cfg)[0]
        assert np.abs(out - want).max() <= TOL, s["material"]
    check_pcm_outputs(subs, pcm_outs, cfg)


@pytest.mark.gpu
def test_mixed_batch_through_reused_slots_device():
    import torch
    import matchering_b200 as mg
    from matchering_b200.batch import master_many
    from matchering_b200.engine import get_plan
    lib = device_lib()
    cfg = mg.Config(fft_size=BATCH_F, max_piece_size=BATCH_PIECE_DEVICE)
    plan = get_plan(cfg)
    depth = 3
    subs, T_MAX, R_MAX = batch_script(plan.layout, depth, BATCH_PIECE_DEVICE)
    alone = [stages_device(cfg, s["t"], s["r"], None) for s in subs]
    check_script_premises(subs, alone, plan.layout, T_MAX, R_MAX, depth)
    wants = [port.main(s["t"].astype(np.float64), s["r"].astype(np.float64), port.config_from(cfg))[0] for s in subs]
    with torch.cuda.device(plan.device):
        outs, states, slots = run_script(Pipe(lib, plan.struct, T_MAX, R_MAX, depth), subs)
        pcm_outs, _, pcm_slots = run_script(Pipe(lib, plan.struct, T_MAX, R_MAX, depth), subs, pcm=True)
    assert [slots.count(k) for k in range(depth)] == [len(s) for s in SLOT_SCRIPTS] and pcm_slots == slots
    worst = 0.0
    for s, a, out, st, want in zip(subs, alone, outs, states, wants):
        ref = state_of(a["state"])
        for f in INT_FIELDS:
            assert getattr(st, f) == getattr(ref, f), (s["material"], s["tkey"], f)
        assert np.isfinite(out).all()
        e = float(np.abs(out - want).max())
        assert e <= TOL, (s["material"], s["tkey"], e)
        worst = max(worst, e)
    worst_pcm = check_pcm_outputs(subs, pcm_outs, cfg)
    # the Python batch entry over the same script, its slot buffers poisoned as well
    lib.mgb_set_option(b"poison_alloc", 1)
    try:
        many = master_many([(s["t"], s["r"]) for s in subs], cfg, depth=3)
    finally:
        lib.mgb_set_option(b"poison_alloc", 0)
    for s, out, want in zip(subs, many, wants):
        e = float(np.abs(out - want).max())
        assert np.isfinite(out).all() and e <= TOL, (s["material"], s["tkey"], e)
        worst = max(worst, e)
    print(f"mixed batch: worst limited output vs oracle {worst:.2e}, PCM {worst_pcm:.2e}")
