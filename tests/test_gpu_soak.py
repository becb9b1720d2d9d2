"""Long and wide GPU parity runs (pytest -m gpu), all through the C ABI.

  * soak: 64 streams x 2000 frames (20 s of audio per stream) x {default, hot, little}, free-running:
      - against the oracle port: PCM and VAD of every stream-frame BIT-EXACT, final network / DSP state bit-exact
        (the port is pinned to the reference build by the CPU suite);
      - against the UNMODIFIED reference, through a sample of its outputs stored in tests/golden/soak_<model>.npz
        (PCM of 4 streams at 48 frames, their VAD at every frame, pitch / silence of 8 traced streams):
        SURVEY App. D rule (ii) -- err(GPU, AVX2 reference) <= 2 * E_ref + floor per quantity, E_ref = |AVX2
        reference - generic-C reference| on the same sample; pitch period and silence flag equal on 100 % of the
        traced non-silent frames; PCM rms error < 1e-3 of the signal rms.
  * wide: 16 384 streams of the little model (BASELINE configs[3]) with 32 spot-checked streams vs the port.
  * conv1 / conv2 memories compared with the port (they were only covered indirectly before).
  * frame-counter wrap: a batch started just below 2^30 (the old mask) and just below the real wrap modulus
    produces the same bits as one started at 0.
  * multi-GPU (needs >= 2 devices, skipped otherwise): the same shard on device 1 == device 0, and a
    rnnoise_batch_create_multi batch over both devices == a single-device batch.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from rnnoise_b200.synth_pcm import batch_pcm, stream_pcm

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SOAK_STREAMS = int(os.environ.get("SOAK_STREAMS", "64"))
SOAK_FRAMES = int(os.environ.get("SOAK_FRAMES", "2000"))
TRACED = 8          # streams whose pitch / silence / gains are traced through the reference's stage functions


@pytest.fixture(scope="module")
def rb():
    import rnnoise_b200
    if not os.path.exists(rnnoise_b200.LIB_PATH):
        from rnnoise_b200 import build
        build.build()
    rnnoise_b200.lib()
    return rnnoise_b200


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def pool_map(fn, items):
    # ctypes releases the GIL inside the C calls, so host threads run the CPU checkers side by side
    with ThreadPoolExecutor(max_workers=max(1, min(32, len(os.sched_getaffinity(0))))) as ex:
        return list(ex.map(fn, items))


def run_port(port, pcm_s):
    """pcm_s [T][480] -> out [T][480], vad [T], final state dict."""
    st = port.create()
    T = pcm_s.shape[0]
    out = np.empty((T, 480), np.float32); vad = np.empty(T, np.float32)
    last = None
    for t in range(T):
        last = port.process_frame(st, pcm_s[t], trace=(t == T - 1))
        out[t] = last["out"]; vad[t] = last["vad"]
    s = st.contents
    fin = dict(lastg=np.array(s.lastg, np.float32), conv1_state=np.array(s.conv1_state, np.float32),
               conv2_state=np.array(s.conv2_state, np.float32), gru=[np.array(s.gru_state[i], np.float32) for i in range(3)],
               pitch=int(s.last_period), pitch_gain=np.float32(s.last_gain), silence=last["silence"])
    port.destroy(st)
    return out, vad, fin


def run_ref(ref, pcm_s, traced):
    st = ref.create()
    T = pcm_s.shape[0]
    out = np.empty((T, 480), np.float32); vad = np.empty(T, np.float32)
    pitch = np.zeros(T, np.int32); sil = np.zeros(T, np.int32)
    for t in range(T):
        if traced:
            r = ref.process_frame_traced(st, pcm_s[t])
            out[t], vad[t], pitch[t], sil[t] = r["out"], r["vad"], r["pitch"], r["silence"]
        else:
            out[t], vad[t] = ref.process_frame(st, pcm_s[t])
    ref.destroy(st)
    return out, vad, pitch, sil


@pytest.mark.parametrize("name", ["default", "hot", "little"])
def test_soak_2000_frames_vs_port_and_live_reference(rb, models_dir, name):
    from oracle.portbind import Port
    S, T = SOAK_STREAMS, SOAK_FRAMES
    mp = os.path.join(models_dir, name + ".bin")
    ids = list(range(S))
    pcm = np.stack([stream_pcm(s, T) for s in ids])                    # [S][T][480]
    model = rb.Model(mp)
    batch = rb.Batch(model, S)
    out, vad = batch.process_frames(pcm.reshape(S, T * 480))          # one multi-frame call: 2000 frames on the GPU
    out = out.reshape(S, T, 480)
    # ---- vs the port: bit-exact on every stream-frame + final state ----
    port = Port(mp)
    res = pool_map(lambda s: run_port(port, pcm[s]), ids)
    for s, (po, pv, fin) in enumerate(res):
        bad = np.nonzero((bits(out[s]) != bits(po)).any(axis=1))[0]
        assert bad.size == 0, f"{name}: stream {s} PCM differs from the port first at frame {bad[0]} (max {np.abs(out[s] - po).max()})"
        assert np.array_equal(bits(vad[s]), bits(pv)), f"{name}: stream {s} VAD differs from the port"
        assert np.array_equal(bits(batch.debug("lastg", s)), bits(fin["lastg"]))
        assert np.array_equal(bits(batch.debug("conv1_state", s)), bits(fin["conv1_state"]))
        g = len(batch.debug("gru1", s)); c2 = batch.debug("conv2_state", s)
        want_u8 = np.array([port.lib.rp_quant_u8(float(x)) for x in fin["conv2_state"][:len(c2)]], np.float32)
        assert np.array_equal(c2, want_u8), f"{name}: conv2 memory of stream {s}"
        for li, k in enumerate(("gru1", "gru2", "gru3")):
            assert np.array_equal(bits(batch.debug(k, s)), bits(fin["gru"][li][:g])), f"{name}: {k} state of stream {s} after {T} frames"
        p = batch.debug("pitch", s)
        assert int(p[0]) == fin["pitch"] and bits(p[1:2])[0] == bits(np.float32([fin["pitch_gain"]]))[0]
    # ---- vs the unmodified reference (SURVEY App. D rule ii), on the sample of its outputs stored by
    # tests/golden/make_golden_soak.py ----
    g = np.load(os.path.join(GOLD, f"soak_{name}.npz"))
    sid, fr, traced = [int(x) for x in g["streams"]], g["frames"], int(g["traced"])
    if T != int(g["frames_total"]) or S <= max(sid + [traced - 1]):
        pytest.skip(f"the stored reference sample covers {int(g['frames_total'])} frames of streams {sid} (port comparison above passed)")
    a_out = np.stack([g[f"s{s}_out"] for s in sid]); g_out = np.stack([g[f"s{s}_generic_out"] for s in sid])
    a_vad = np.stack([g[f"s{s}_vad"] for s in sid]); g_vad = np.stack([g[f"s{s}_generic_vad"] for s in sid])
    e_ref_pcm, e_ref_vad = np.abs(a_out - g_out), np.abs(a_vad - g_vad)
    err_pcm, err_vad = np.abs(out[sid][:, fr] - a_out), np.abs(vad[sid] - a_vad)
    rms = lambda x: float(np.sqrt(np.mean(np.square(x, dtype=np.float64))))
    report = dict(pcm_max=float(err_pcm.max()), pcm_rms=rms(err_pcm), e_ref_pcm_max=float(e_ref_pcm.max()), e_ref_pcm_rms=rms(e_ref_pcm),
                  vad_max=float(err_vad.max()), e_ref_vad_max=float(e_ref_vad.max()), signal_rms=rms(a_out))
    print(name, "soak vs reference:", report)
    assert report["pcm_max"] <= 2 * report["e_ref_pcm_max"] + 0.25, report
    assert report["pcm_rms"] <= 2 * report["e_ref_pcm_rms"] + 0.02, report
    assert report["vad_max"] <= 2 * report["e_ref_vad_max"] + 2e-4, report
    # "never worse than PCM rms 1e-3 of the signal rms" (App. D) -- unless the reference's own two builds already differ
    # by more than that for this model (the 'hot' model: E_ref rms = 1.8e-3 of the signal), where 2 * E_ref governs
    assert report["pcm_rms"] <= max(1e-3 * report["signal_rms"], 2 * report["e_ref_pcm_rms"]), report
    # pitch period / silence flag on the traced streams: GPU values are those of the port (bit-exact chain above);
    # the port's trace is compared with the reference's stage functions frame by frame
    def port_trace(s):
        st = port.create(); p = np.zeros(T, np.int32); q = np.zeros(T, np.int32)
        for t in range(T):
            r = port.process_frame(st, pcm[s, t]); p[t], q[t] = r["pitch"], r["silence"]
        port.destroy(st)
        return p, q
    pt = pool_map(port_trace, list(range(traced)))
    nonsilent = 0
    for s, (p, q) in enumerate(pt):
        ref_pitch, ref_sil = g[f"s{s}_pitch"].astype(np.int32), g[f"s{s}_silence"].astype(np.int32)
        assert np.array_equal(q, ref_sil), f"{name}: silence flags of stream {s}"
        live = ref_sil == 0
        nonsilent += int(live.sum())
        assert np.array_equal(p[live], ref_pitch[live]), f"{name}: pitch period of stream {s} on non-silent frames"
    assert nonsilent > 0.5 * traced * T
    batch.destroy(); model.free()


def test_little_model_16384_streams_spot_checked(rb, models_dir):
    """BASELINE configs[3]: 'little' model, 16 384 streams on one GPU; 32 streams spread over the batch (tile
    edges, lane edges, last stream) bit-exact against the port for 40 frames."""
    from oracle.portbind import Port
    S, T, P = 16384, 40, 128
    mp = os.path.join(models_dir, "little.bin")
    base = batch_pcm(P, T)                                   # [T][P][480]; stream s of the batch = pool stream s % P
    model = rb.Model(mp); batch = rb.Batch(model, S)
    port = Port(mp)
    rng = np.random.default_rng(5)
    check = sorted({0, 1, 127, 128, 2047, 2048, 8191, 8192, 8193, 12287, 16383, 16256} | set(int(x) for x in rng.integers(0, S, 20)))
    assert len(check) >= 32
    want = {p: run_port(port, base[:, p]) for p in sorted({s % P for s in check})}
    outs = np.empty((T, len(check), 480), np.float32); vads = np.empty((T, len(check)), np.float32)
    for t in range(T):
        out, vad = batch.process(np.ascontiguousarray(np.tile(base[t], (S // P, 1))))
        outs[t] = out[check]; vads[t] = vad[check]
    for i, s in enumerate(check):
        po, pv, fin = want[s % P]
        assert np.array_equal(bits(outs[:, i]), bits(po)), f"stream {s}"
        assert np.array_equal(bits(vads[:, i]), bits(pv)), f"stream {s}"
        for li, k in enumerate(("gru1", "gru2", "gru3")):
            assert np.array_equal(bits(batch.debug(k, s)), bits(fin["gru"][li][:384])), (k, s)
    batch.destroy(); model.free()


@pytest.mark.parametrize("start", [(1 << 30) - 3, (18 << 24) - 3, (1 << 40) + 5])
def test_frame_counter_wrap_is_seamless(rb, models_dir, start):
    """ADVICE/VERDICT r1: parity, spectrum slot and ring base come from the frame counter; a batch whose counter
    starts just below 2^30 (the old mask) / just below the wrap modulus 18 << 24 / far beyond must produce the
    bits of a batch started at 0 across the boundary."""
    mp = os.path.join(models_dir, "default.bin")
    ids, T = [0, 3, 15, 40, 7], 14
    pcm = np.stack([stream_pcm(s, T) for s in ids], axis=1)
    model = rb.Model(mp)
    a, b = rb.Batch(model, len(ids)), rb.Batch(model, len(ids))
    b.debug_set_frame_counter(start)
    for t in range(T):
        oa, va = a.process(pcm[t]); ob, vb = b.process(pcm[t])
        assert np.array_equal(bits(oa), bits(ob)) and np.array_equal(bits(va), bits(vb)), f"frame {t} (counter {start + t})"
        for i in range(len(ids)):
            for k in ("features", "X", "P", "Ex", "gru3", "pitch"):
                assert np.array_equal(bits(a.debug(k, i)), bits(b.debug(k, i))), (k, t, i)
    a.destroy(); b.destroy(); model.free()


def test_conv_memories_match_port(rb, port_default, models_dir):
    """conv1 memory (fp32) and conv2 memory (kept as the u8 operand the int8 GEMM consumes) against the port's
    float memories, every frame, including streams with silent frames (memories must freeze there)."""
    mp = os.path.join(models_dir, "default.bin")
    ids, T = [15, 31, 2, 9], 60
    pcm = np.stack([stream_pcm(s, T) for s in ids], axis=1)
    model = rb.Model(mp); batch = rb.Batch(model, len(ids))
    states = [port_default.create() for _ in ids]
    q = port_default.lib.rp_quant_u8
    silent_seen = 0
    for t in range(T):
        batch.process(pcm[t])
        for i in range(len(ids)):
            r = port_default.process_frame(states[i], pcm[t, i])
            silent_seen += r["silence"]
            st = states[i].contents
            assert np.array_equal(bits(batch.debug("conv1_state", i)), bits(np.array(st.conv1_state, np.float32))), (t, ids[i])
            c2 = batch.debug("conv2_state", i)
            want = np.array([q(float(x)) for x in np.array(st.conv2_state, np.float32)[:len(c2)]], np.float32)
            assert np.array_equal(c2, want), (t, ids[i])
    assert silent_seen > 0
    for st in states:
        port_default.destroy(st)
    batch.destroy(); model.free()


def _ndev():
    import ctypes as C
    try:
        rt = C.CDLL("libcudart.so")
    except OSError:
        import torch
        return torch.cuda.device_count()
    n = C.c_int(0)
    return n.value if rt.cudaGetDeviceCount(C.byref(n)) == 0 else 0


def test_second_device_and_multi_device_batch_equal_single_device(rb, models_dir):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    mp = os.path.join(models_dir, "default.bin")
    S, T = 2304, 12                       # two lanes per device in the multi-device batch
    base = batch_pcm(96, T)
    pcm = np.ascontiguousarray(np.tile(base, (1, S // 96, 1)))
    model = rb.Model(mp)
    b0 = rb.Batch(model, S, 0)
    b1 = rb.Batch(model, S, 1)
    bm = rb.Batch(model, S, devices=[0, 1])
    assert bm.nb_devices == 2 and bm.shard(0) == (0, 0, S // 2) and bm.shard(1) == (1, S // 2, S // 2)
    # device-pointer multi call: per-device shard buffers
    d_in = [torch.empty(S // 2, 480, device=f"cuda:{k}") for k in range(2)]
    d_out = [torch.empty_like(x) for x in d_in]
    d_vad = [torch.empty(S // 2, device=f"cuda:{k}") for k in range(2)]
    bd = rb.Batch(model, S, devices=[0, 1])
    for t in range(T):
        o0, v0 = b0.process(pcm[t]); o1, v1 = b1.process(pcm[t]); om, vm = bm.process(pcm[t])
        assert np.array_equal(bits(o0), bits(o1)) and np.array_equal(bits(v0), bits(v1)), f"device 1 != device 0, frame {t}"
        assert np.array_equal(bits(o0), bits(om)) and np.array_equal(bits(v0), bits(vm)), f"multi-device batch, frame {t}"
        for k in range(2):
            d_in[k].copy_(torch.from_numpy(pcm[t, k * S // 2:(k + 1) * S // 2]))
            torch.cuda.synchronize(k)
        bd.process_device_multi([x.data_ptr() for x in d_out], [x.data_ptr() for x in d_in], [x.data_ptr() for x in d_vad])
        bd.sync()
        od = np.concatenate([x.cpu().numpy() for x in d_out]); vd = np.concatenate([x.cpu().numpy() for x in d_vad])
        assert np.array_equal(bits(o0), bits(od)) and np.array_equal(bits(v0), bits(vd)), f"device-pointer multi call, frame {t}"
    for b in (b0, b1, bm, bd):
        b.destroy()
    model.free()
