"""The GPU's per-stream DSP source (rnnoise_b200/csrc/dsp_stream.cuh) executed on the host, thread id
by thread id, must be BIT-IDENTICAL to the oracle port (hence to the reference build): checks the
indexing, work partitioning and arithmetic of the exact code the GPU runs, without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.portbind import Port, fptr
from rnnoise_b200.synth_pcm import stream_pcm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "emu_dsp.cpp")
EMU_SO = os.path.join(ROOT, "tests", "emu", "libemu_dsp.so")


@pytest.fixture(scope="module")
def emu():
    deps = [EMU_SRC] + [os.path.join(ROOT, "rnnoise_b200", "csrc", f) for f in ("dsp_core.cuh", "dsp_stream.cuh", "dsp_pitch.cuh", "dsp_tables.hpp")]
    if not os.path.exists(EMU_SO) or any(os.path.getmtime(d) > os.path.getmtime(EMU_SO) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DPITCH_NS=4",
                        "-I", os.path.join(ROOT, "rnnoise_b200", "csrc"), EMU_SRC, "-o", EMU_SO], check=True)
    E = C.CDLL(EMU_SO)
    E.emu_create.restype = C.c_void_p
    E.emu_destroy.argtypes = [C.c_void_p]
    E.emu_analysis.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
    E.emu_get.argtypes = [C.c_void_p, C.c_int] + [C.POINTER(C.c_float)] * 6
    E.emu_synthesis.argtypes = [C.c_void_p, C.c_int] + [C.POINTER(C.c_float)] * 3
    E.emu_advance.argtypes = [C.c_void_p]
    E.emu_group_create.restype = C.c_void_p
    E.emu_group_destroy.argtypes = [C.c_void_p]
    E.emu_group_analysis.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int)]
    return E


@pytest.mark.parametrize("streams,frames", [((0, 15, 7, 3), 60), ((5, 31, 2), 40), ((9,), 30)])
def test_device_dsp_source_is_bit_identical_to_port(emu, port_default, streams, frames):
    """Groups of up to PITCH_NS streams share one emulated pitch CTA (packed serial chains); partial
    groups exercise the absent-stream guards."""
    assert emu.emu_streams() >= len(streams)
    pcm = np.stack([stream_pcm(s, frames) for s in streams], axis=1)   # [frames][n][480]
    states = [port_default.create() for _ in streams]
    e = emu.emu_create()
    for f in range(frames):
        emu.emu_analysis(e, fptr(np.ascontiguousarray(pcm[f])), len(streams))
        for q, s in enumerate(streams):
            b = port_default.process_frame(states[q], pcm[f, q])
            xb = np.zeros(480, np.float32); feat = np.zeros(65, np.float32)
            X = np.zeros(962, np.float32); P = np.zeros(962, np.float32)
            bands = np.zeros(96, np.float32); pitch = np.zeros(2, np.float32)
            sil = emu.emu_get(e, q, fptr(xb), fptr(feat), fptr(X), fptr(P), fptr(bands), fptr(pitch))
            out = np.zeros(480, np.float32); lastg = np.zeros(32, np.float32)
            emu.emu_synthesis(e, q, fptr(b["g_raw"]), fptr(out), fptr(lastg))
            for k, u, v in (("xb", xb, b["xb"]), ("features", feat, b["features"]), ("X", X, b["X"]), ("P", P, b["P"]),
                            ("Ex", bands[:32], b["Ex"]), ("Ep", bands[32:64], b["Ep"]), ("Exp", bands[64:], b["Exp"]),
                            ("out", out, b["out"]), ("lastg", lastg, b["lastg"])):
                assert u.tobytes() == v.tobytes(), (k, f, s)
            assert sil == b["silence"] and int(pitch[0]) == b["pitch"], (f, s)
            assert pitch[1:].tobytes() == np.float32(b["pitch_gain"]).tobytes()
        emu.emu_advance(e)
    emu.emu_destroy(e)
    for st in states:
        port_default.destroy(st)


def test_remove_doubling_candidates_exact_over_whole_domain(emu):
    """rd_candidate() replaces the reference's integer divisions (pitch.c:462-481) by float multiply +
    truncate and its second_check[] table by arithmetic: every (k, T0) must give the reference's integers."""
    second_check = [0, 0, 3, 2, 3, 2, 5, 2, 3, 2, 3, 2, 5, 2, 3, 2]
    t1, t1b = C.c_int(), C.c_int()
    emu.emu_rd_candidate.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    for k in range(1, 16):
        for T0 in range(0, 385):
            emu.emu_rd_candidate(k, T0, C.byref(t1), C.byref(t1b))
            if k == 1:
                want = (T0, T0)
            else:
                w1 = (2 * T0 + k) // (2 * k)
                want = (w1, (T0 if w1 + T0 > 384 else T0 + w1) if k == 2 else (2 * second_check[k] * T0 + k) // (2 * k))
            assert (t1.value, t1b.value) == want, (k, T0)


@pytest.mark.parametrize("first,n,frames", [(0, 16, 80), (16, 16, 40), (40, 5, 40), (15, 1, 150), (100, 11, 30)])
def test_pitch_group_kernel_source_is_bit_identical_to_port(emu, port_default, first, n, frames):
    """The default pitch kernel's body (dsp_pitch.cuh: PG streams per CTA, home warps + chain warps, refinement
    correlations after the decision) executed thread id by thread id: pitch period, pitch gain, silence flag and
    all 65 features (which carry the pitch-lagged spectrum) must equal the port's bits; full and partial groups,
    streams with digital silence (every 16th), 150-frame run for the continuity prior."""
    assert emu.emu_group_streams() >= n
    ids = list(range(first, first + n))
    pcm = np.stack([stream_pcm(s, frames) for s in ids], axis=1)
    states = [port_default.create() for _ in ids]
    e = emu.emu_group_create()
    feat = np.zeros((n, 65), np.float32); pitch = np.zeros((n, 2), np.float32); sil = np.zeros(n, np.int32)
    for f in range(frames):
        emu.emu_group_analysis(e, fptr(np.ascontiguousarray(pcm[f])), n, fptr(feat), fptr(pitch), sil.ctypes.data_as(C.POINTER(C.c_int)))
        for q, s in enumerate(ids):
            b = port_default.process_frame(states[q], pcm[f, q])
            assert int(pitch[q, 0]) == b["pitch"], (f, s, int(pitch[q, 0]), b["pitch"])
            assert pitch[q, 1:].tobytes() == np.float32(b["pitch_gain"]).tobytes(), (f, s)
            assert sil[q] == b["silence"], (f, s)
            assert feat[q].tobytes() == b["features"].tobytes(), (f, s)
    emu.emu_group_destroy(e)
    for st in states:
        port_default.destroy(st)


def test_log_energy_follower_in_float_equals_the_reference_double_form():
    """spectrum_stream runs the floor follower of denoise.c:380-387 in float (dsp_stream.cuh); the reference evaluates
    follow - 1.5 and the maxima in double.  Both forms over 200k random band vectors, ties and near-ties included."""
    rng = np.random.default_rng(5)
    n = 200_000
    ly = rng.uniform(-2.2, 9.0, size=(n, 32)).astype(np.float32)
    # near-ties: a band exactly 1.5 (or 7) below its predecessor / the running maximum, +- one ulp
    k = rng.integers(1, 32, size=n)
    rows = np.arange(n)
    tie = ly[rows, k - 1] - np.float32(1.5)
    ly[rows, k] = np.where(rows % 3 == 0, tie, np.where(rows % 3 == 1, np.nextafter(tie, np.float32(np.inf)), ly[rows, k]))
    with np.errstate(invalid="ignore"):
        def run(double_form):
            out = np.empty_like(ly)
            logmax = np.full(n, -2, np.float32); follow = np.full(n, -2, np.float32)
            for i in range(32):
                if double_form:
                    f15 = follow.astype(np.float64) - 1.5
                    m1 = np.where(f15 > ly[:, i], f15, ly[:, i].astype(np.float64))
                    lm7 = (logmax - np.float32(7)).astype(np.float32)
                    v = np.where(lm7 > m1, lm7.astype(np.float64), m1).astype(np.float32)
                    logmax = np.where(logmax > v, logmax, v)
                    follow = np.where(f15 > v, f15, v.astype(np.float64)).astype(np.float32)
                else:
                    f15 = (follow - np.float32(1.5)).astype(np.float32)
                    m1 = np.where(f15 > ly[:, i], f15, ly[:, i])
                    lm7 = (logmax - np.float32(7)).astype(np.float32)
                    v = np.where(lm7 > m1, lm7, m1)
                    logmax = np.where(logmax > v, logmax, v)
                    follow = np.where(f15 > v, f15, v)
                out[:, i] = v
            return out
        a, b = run(True), run(False)
    assert a.tobytes() == b.tobytes()


def test_fft_buffer_swizzle_is_a_block_permutation_without_bank_conflicts(emu):
    """dsp_core.cuh `fsw`: a permutation (involution) of every aligned block of 16 complex elements under which every
    FFT stage's half warp (16 lanes x 8-byte elements = one shared-memory wavefront) touches 16 different bank pairs --
    and the radix-4 m = 4 stage, unswizzled, only 4 (the conflict the swizzle removes)."""
    f = [emu.emu_fsw(i) for i in range(960)]
    assert sorted(f) == list(range(960))
    assert all(f[f[i]] == i and f[i] // 16 == i // 16 for i in range(960))

    def banks(idx):          # 8-byte elements: 16 bank pairs
        return {i % 16 for i in idx}

    for b0 in range(0, 240, 16):                      # radix-4 stages: butterfly b = 16 consecutive lanes
        for q in range(4):
            m4 = [16 * (b // 4) + b % 4 + 4 * q for b in range(b0, b0 + 16)]
            assert len(banks(m4)) == 4                 # the unswizzled layout: 4-way conflict
            assert len(banks(f[i] for i in m4)) == 16
            m16 = [64 * (b // 16) + b % 16 + 16 * q for b in range(b0, b0 + 16)]
            assert len(banks(f[i] for i in m16)) == 16
    for b0 in range(0, 320, 16):                      # radix 3: m = 64
        for q in range(3):
            assert len(banks(f[192 * (b // 64) + b % 64 + 64 * q] for b in range(b0, b0 + 16))) == 16
    for u0 in range(0, 192, 16):                      # radix 5: m = 192
        for q in range(5):
            assert len(banks(f[u + 192 * q] for u in range(u0, u0 + 16))) == 16
    for i0 in range(0, 480, 16):                      # linear consumers (spectrum stores, per-bin terms)
        assert len(banks(f[i] for i in range(i0, i0 + 16))) == 16
    for g0 in range(0, 240, 4):                       # stage 1 writes 4 contiguous elements per group
        for g in range(g0, g0 + 4):
            assert [f[4 * g + q] for q in range(4)] == list(range(f[4 * g], f[4 * g] + 4))


def _edge_signals(frames):
    n = frames * 480
    t = np.arange(n)
    rng = np.random.default_rng(1)
    yield "fullscale_square", (32767 * np.sign(np.sin(2 * np.pi * 440 * t / 48000))).astype(np.float32)
    x = np.zeros(n, np.float32); x[::997] = 30000
    yield "impulses", x
    yield "dc", np.full(n, 12345.0, np.float32)
    yield "tiny_noise", (rng.standard_normal(n) * 1e-30).astype(np.float32)
    yield "denormal_noise", (rng.standard_normal(n) * 1e-41).astype(np.float32)
    yield "clipping_noise", np.clip(rng.standard_normal(n) * 40000, -32768, 32767).astype(np.float32)
    x = (rng.standard_normal(n) * 3000).astype(np.float32); x[5000:5480] = 0; x[9600:14400] = 0
    yield "gaps_of_silence", x
    x = (rng.standard_normal(n) * 3000).astype(np.float32); x[7000] = np.nan
    yield "one_nan", x
    x = (rng.standard_normal(n) * 3000).astype(np.float32); x[7000] = np.inf
    yield "one_inf", x


@pytest.mark.parametrize("name,sig", list(_edge_signals(40)), ids=[n for n, _ in _edge_signals(40)])
def test_device_dsp_source_on_edge_case_signals(emu, port_default, name, sig):
    """Full-scale, impulsive, constant, vanishing (incl. denormal), clipped and gapped input: the device DSP source stays
    bit-identical to the port.  A non-finite sample poisons the state of the reference for good (every later output sample is
    NaN); the device source does the same, sample for sample -- only the sign bit of those NaNs (which operand of a
    commutative x86 instruction came first) is outside the contract."""
    frames = len(sig) // 480
    pcm = sig.reshape(frames, 480)
    st = port_default.create()
    e = emu.emu_create()
    finite = np.isfinite(sig).all()
    for f in range(frames):
        emu.emu_analysis(e, fptr(np.ascontiguousarray(pcm[f][None])), 1)
        b = port_default.process_frame(st, pcm[f])
        xb = np.zeros(480, np.float32); feat = np.zeros(65, np.float32)
        X = np.zeros(962, np.float32); P = np.zeros(962, np.float32)
        bands = np.zeros(96, np.float32); pitch = np.zeros(2, np.float32)
        sil = emu.emu_get(e, 0, fptr(xb), fptr(feat), fptr(X), fptr(P), fptr(bands), fptr(pitch))
        out = np.zeros(480, np.float32); lastg = np.zeros(32, np.float32)
        emu.emu_synthesis(e, 0, fptr(b["g_raw"]), fptr(out), fptr(lastg))
        for k, u, v in (("xb", xb, b["xb"]), ("features", feat, b["features"]), ("X", X, b["X"]), ("P", P, b["P"]),
                        ("Ex", bands[:32], b["Ex"]), ("Ep", bands[32:64], b["Ep"]), ("Exp", bands[64:], b["Exp"]),
                        ("out", out, b["out"]), ("lastg", lastg, b["lastg"])):
            if finite:
                assert u.tobytes() == v.tobytes(), (name, k, f)
            else:
                assert np.array_equal(np.isnan(u), np.isnan(v)), (name, k, f)
                m = ~np.isnan(u)
                assert u[m].tobytes() == v[m].tobytes(), (name, k, f)
        if finite:
            assert sil == b["silence"] and int(pitch[0]) == b["pitch"], (name, f)
        emu.emu_advance(e)
    emu.emu_destroy(e)
