"""GPU parity tests (run on an H100: pytest -m gpu).  Everything goes through the C ABI of
include/rnnoise.h (ctypes); the checker is the oracle port (bit-pinned to the reference build by
tests/test_oracle_port.py) plus the committed reference goldens.

Bars (DESIGN.md "Parity"):
  * DSP quantities (biquad output, X, P, Ex, Ep, Exp, features, pitch period, silence flag): bit-exact.
  * int8 accumulators: exact by construction; network outputs (gains, VAD, states) and PCM: the CUDA
    path implements the port's arithmetic operation for operation, so they are compared bit-exact
    against the port as well, and against the REFERENCE goldens within the reference's own
    cross-build envelope: err <= 2 * E_ref + floor, E_ref = |AVX2 build - generic-C build|.
"""
import os

import numpy as np
import pytest

from rnnoise_b200.synth_pcm import batch_pcm, stream_pcm

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


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


def compare_with_port(rb, port, model_path, stream_ids, frames, exact_nn=True):
    model = rb.Model(model_path)
    S = len(stream_ids)
    batch = rb.Batch(model, S)
    pcm = np.stack([stream_pcm(s, frames) for s in stream_ids], axis=1)  # [frames][S][480]
    states = [port.create() for _ in stream_ids]
    worst = {}
    for f in range(frames):
        out, vad = batch.process(pcm[f])
        for i in range(S):
            r = port.process_frame(states[i], pcm[f, i])
            tag = f"frame {f} stream {stream_ids[i]}"
            assert int(batch.debug("silence", i)[0]) == r["silence"], tag
            assert int(batch.debug("pitch", i)[0]) == r["pitch"], tag
            for key, pk in (("xb", "xb"), ("X", "X"), ("P", "P"), ("Ex", "Ex"), ("Ep", "Ep"), ("Exp", "Exp"),
                            ("features", "features")):
                assert np.array_equal(bits(batch.debug(key, i)), bits(r[pk])), f"{key} not bit-exact, {tag}"
            nn = dict(out=(out[i], r["out"]), vad=(vad[i:i + 1], np.float32([r["vad"]])), lastg=(batch.debug("lastg", i), r["lastg"]))
            if not r["silence"]:
                nn["gains"] = (batch.debug("gains", i), r["g_raw"])
            for k, (u, v) in nn.items():
                d = float(np.abs(np.asarray(u, np.float64) - np.asarray(v, np.float64)).max())
                worst[k] = max(worst.get(k, 0.0), d)
                if exact_nn:
                    assert np.array_equal(bits(u), bits(v)), f"{k} differs from the port by {d}, {tag}"
            st = states[i].contents
            for li, k in enumerate(("gru1", "gru2", "gru3")):
                g = np.array(st.gru_state[li][:len(batch.debug(k, i))], np.float32)
                if exact_nn:
                    assert np.array_equal(bits(batch.debug(k, i)), bits(g)), f"{k} state, {tag}"
    for st in states:
        port.destroy(st)
    batch.destroy()
    model.free()
    return worst


def test_default_model_bit_exact_vs_port(rb, port_default, models_dir):
    ids = [0, 1, 2, 3, 15, 7, 31, 100, 47]
    worst = compare_with_port(rb, port_default, os.path.join(models_dir, "default.bin"), ids, 70)
    print("max |gpu - port|:", worst)


@pytest.mark.parametrize("name", ["hot", "little", "g256", "tiny", "little_b"])
@pytest.mark.parametrize("net", ["fused", "layers"])
def test_other_models_bit_exact_vs_port(rb, models_dir, name, net, monkeypatch):
    """Model matrix x both network paths (the fused cluster kernel is the default for small batches, one launch per
    layer for large ones): tiny (cond 96) and little_b (GRU 192) exercise the zero-weight padding of the contraction
    rows to the 128-byte swizzle atom, g256 / little_b / tiny other unit splits."""
    from oracle.portbind import Port
    monkeypatch.setenv("RNNOISE_B200_NET_KERNEL", net)
    port = Port(os.path.join(models_dir, name + ".bin"))
    worst = compare_with_port(rb, port, os.path.join(models_dir, name + ".bin"), [0, 15, 5], 50 if net == "fused" else 30)
    print(name, net, "max |gpu - port|:", worst)


@pytest.mark.parametrize("name", ["default", "hot", "little"])
def test_against_reference_goldens(rb, models_dir, name):
    """Committed outputs of the unmodified reference (AVX2 path): DSP bit-exact, network/PCM inside
    2x the reference's own AVX2-vs-generic-C envelope."""
    g = np.load(os.path.join(GOLD, f"ref_{name}.npz"))
    frames, ids = int(g["frames"]), [int(s) for s in g["streams"]]
    model = rb.Model(os.path.join(models_dir, name + ".bin"))
    batch = rb.Batch(model, len(ids))
    pcm = np.stack([stream_pcm(s, frames) for s in ids], axis=1)
    got = {k: np.zeros((frames, len(ids)) + shp, np.float32) for k, shp in
           (("features", (65,)), ("Ex", (32,)), ("g_raw", (32,)), ("out", (480,)), ("lastg", (32,)), ("vad", ()), ("pitch", ()), ("silence", ()))}
    for f in range(frames):
        out, vad = batch.process(pcm[f])
        got["out"][f], got["vad"][f] = out, vad
        for i in range(len(ids)):
            got["features"][f, i] = batch.debug("features", i); got["Ex"][f, i] = batch.debug("Ex", i)
            got["lastg"][f, i] = batch.debug("lastg", i)
            got["pitch"][f, i] = batch.debug("pitch", i)[0]; got["silence"][f, i] = batch.debug("silence", i)[0]
            got["g_raw"][f, i] = 0 if got["silence"][f, i] else batch.debug("gains", i)
    for i, s in enumerate(ids):
        assert np.array_equal(bits(got["features"][:, i]), bits(g[f"s{s}_features"])), f"features vs reference, stream {s}"
        assert np.array_equal(bits(got["Ex"][:, i]), bits(g[f"s{s}_Ex"]))
        assert np.array_equal(got["pitch"][:, i].astype(int), g[f"s{s}_pitch"])
        assert np.array_equal(got["silence"][:, i].astype(int), g[f"s{s}_silence"])
        for key, floor in (("g_raw", 2e-4), ("vad", 2e-4), ("lastg", 2e-4), ("out", 0.25)):
            ref = g[f"s{s}_{key}"].reshape(got[key][:, i].shape)
            e_ref = float(np.abs(g[f"s{s}_generic_{key}"].reshape(ref.shape) - ref).max())
            err = float(np.abs(got[key][:, i] - ref).max())
            assert err <= 2 * e_ref + floor, (name, s, key, err, e_ref)
    batch.destroy(); model.free()


def test_single_stream_api_equals_batch(rb, models_dir):
    """rnnoise_create()/rnnoise_process_frame() (reference surface, in == out aliasing as in
    examples/rnnoise_demo.c:57) gives exactly what the batched call gives for the same stream."""
    import ctypes as C
    L = rb.lib()
    mp = os.path.join(models_dir, "default.bin")
    model = rb.Model(mp)
    st = L.rnnoise_create(model.handle)
    assert st
    batch = rb.Batch(model, 3)
    frames = 25
    pcm = np.stack([stream_pcm(s, frames) for s in (4, 5, 6)], axis=1)
    for f in range(frames):
        out, vad = batch.process(pcm[f])
        x = pcm[f, 1].copy()
        p = x.ctypes.data_as(C.POINTER(C.c_float))
        v = L.rnnoise_process_frame(st, p, p)
        assert np.array_equal(bits(x), bits(out[1])) and np.float32(v) == vad[1]
    L.rnnoise_destroy(st)
    batch.destroy(); model.free()


def test_streams_are_independent_and_reset_works(rb, models_dir):
    """Same input on every stream -> identical output on every stream (no cross-stream term), and a
    reset stream restarts exactly like a fresh state."""
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 300, 12   # S not a multiple of any tile size used by the kernels
    batch = rb.Batch(model, S)
    one = stream_pcm(9, 2 * frames)
    first = []
    for f in range(frames):
        out, vad = batch.process(np.repeat(one[f][None], S, 0))
        assert np.array_equal(bits(out), np.repeat(bits(out[:1]), S, 0)) and np.all(vad == vad[0])
        first.append(out[0].copy())
    batch.reset_stream(137)
    for f in range(frames):   # replay the same frames on the reset stream only
        x = np.repeat(one[frames + f][None], S, 0)
        x[137] = one[f]
        out, _ = batch.process(x)
        assert np.array_equal(bits(out[137]), bits(first[f])), f
    batch.destroy(); model.free()


def test_device_pointer_call_in_place(rb, models_dir):
    """Device-buffer entry point with d_out aliasing d_in, driven from torch-allocated memory."""
    import torch
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 64, 6
    a, b = rb.Batch(model, S), rb.Batch(model, S)
    pcm = batch_pcm(S, frames)
    for f in range(frames):
        ref_out, ref_vad = a.process(pcm[f])
        d = torch.from_numpy(pcm[f]).cuda()
        dv = torch.empty(S, device="cuda")
        torch.cuda.synchronize()
        b.process_device(d.data_ptr(), d.data_ptr(), dv.data_ptr())
        b.sync()
        assert np.array_equal(bits(d.cpu().numpy()), bits(ref_out)) and np.array_equal(dv.cpu().numpy(), ref_vad)
    a.destroy(); b.destroy(); model.free()


def test_full_size_properties_4096_streams(rb, models_dir):
    """BASELINE config[1] size: 4096 streams.  Size-independent properties: streams fed zeros stay
    exactly silent (VAD 0, output 0), duplicated streams stay bit-identical, and a spot-checked
    stream equals the port."""
    from oracle.portbind import Port
    S, frames = 4096, 8
    mp = os.path.join(models_dir, "default.bin")
    model = rb.Model(mp)
    batch = rb.Batch(model, S)
    base = batch_pcm(64, frames)                       # 64 distinct streams, tiled 64x
    port = Port(mp); st = port.create()
    for f in range(frames):
        x = np.tile(base[f], (S // 64, 1))
        x[1::128] = 0.0                                # some all-zero streams
        out, vad = batch.process(x)
        assert np.array_equal(bits(out[:64][2::2]), bits(out[64 * 17:64 * 18][2::2]))
        assert not out[1::128].any() and not vad[1::128].any()
        r = port.process_frame(st, base[f, 5])
        assert np.array_equal(bits(out[64 * 40 + 5]), bits(r["out"])) and np.float32(r["vad"]) == vad[64 * 40 + 5]
    batch.destroy(); model.free()


def test_gru_tensor_core_paths_equal_dp4a_path(rb, models_dir):
    """The wgmma GRU kernels (u8 x s8 -> s32 in registers; tc2 = persistent pipelined default, tc1 = one tile
    per CTA) and the CUDA-core dp4a kernel accumulate the same exact integers, so whole-pipeline outputs
    and GRU states must be bit-identical; S = 300 exercises a partial 128-row tile (TMA zero fill + guards)."""
    model = rb.Model(os.path.join(models_dir, "hot.bin"))
    S, frames = 300, 10
    batches = {}
    for mode in ("dp4a", "tc1", "tc2"):
        os.environ["RNNOISE_B200_GRU_KERNEL"] = mode
        batches[mode] = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_GRU_KERNEL"]
    pcm = batch_pcm(S, frames)
    for f in range(frames):
        res = {m: b.process(pcm[f]) for m, b in batches.items()}
        for m in ("tc1", "tc2"):
            assert np.array_equal(bits(res[m][0]), bits(res["dp4a"][0])) and np.array_equal(bits(res[m][1]), bits(res["dp4a"][1])), (m, f)
            for s in (0, 127, 128, 255, 256, 299):
                for k in ("gru1", "gru2", "gru3", "gains"):
                    assert np.array_equal(bits(batches[m].debug(k, s)), bits(batches["dp4a"].debug(k, s))), (m, k, s, f)
    for b in batches.values():
        b.destroy()
    # conv2: tensor-core kernel (default) vs dp4a kernel
    os.environ["RNNOISE_B200_CONV2_KERNEL"] = "dp4a"
    a = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_CONV2_KERNEL"]
    b = rb.Batch(model, S)
    for f in range(frames):
        oa, va = a.process(pcm[f]); ob, vb = b.process(pcm[f])
        assert np.array_equal(bits(oa), bits(ob)) and np.array_equal(bits(va), bits(vb)), f
        for s in (0, 128, 299):
            for k in ("conv2_out", "conv2_state", "gru3"):
                assert np.array_equal(bits(a.debug(k, s)), bits(b.debug(k, s))), (k, s, f)
    a.destroy(); b.destroy()
    # output heads: register-tiled bulk-copy kernel (default) vs the cp.async kernel; S = 300 leaves a partial tile
    os.environ["RNNOISE_B200_HEADS_KERNEL"] = "cpasync"
    a = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_HEADS_KERNEL"]
    tiles = {}
    for t in ("8", "16", "32", "32w"):    # streams per CTA of the register-tiled kernel (1, 2 or 4 streams per thread on 4 compute warps; 2 on 8)
        os.environ["RNNOISE_B200_HEADS_TILE"] = t
        tiles[t] = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_HEADS_TILE"]
    for f in range(frames):
        oa, va = a.process(pcm[f])
        for t, b in tiles.items():
            ob, vb = b.process(pcm[f])
            assert np.array_equal(bits(oa), bits(ob)) and np.array_equal(bits(va), bits(vb)), (t, f)
            for s in (0, 7, 8, 31, 32, 288, 295, 296, 299):
                assert np.array_equal(bits(a.debug("gains", s)), bits(b.debug("gains", s))), (t, s, f)
    a.destroy()
    for b in tiles.values():
        b.destroy()
    # network: one fused cluster kernel for conv1 + conv2 + 3 GRU layers (default) vs the same without the conv1
    # prologue vs one launch per layer
    os.environ["RNNOISE_B200_NET_KERNEL"] = "layers"
    a = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_NET_KERNEL"]
    os.environ["RNNOISE_B200_NET_KERNEL"] = "fused"
    os.environ["RNNOISE_B200_NET_CLUSTER"] = "4"
    os.environ["RNNOISE_B200_NET_CONV1"] = "0"
    c = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_NET_CONV1"]
    b = rb.Batch(model, S)
    os.environ["RNNOISE_B200_NET_CLUSTER"] = "8"
    d = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_NET_CLUSTER"]
    del os.environ["RNNOISE_B200_NET_KERNEL"]
    assert (a.launches_per_frame, c.launches_per_frame, b.launches_per_frame) == (10, 7, 6)
    for f in range(2 * frames):
        x = pcm[f % frames]
        oa, va = a.process(x); oc, vc = c.process(x); ob, vb = b.process(x); od, vd = d.process(x)
        assert np.array_equal(bits(oa), bits(od)) and np.array_equal(bits(va), bits(vd)), ("8-CTA clusters", f)
        for s in (0, 31, 32, 127, 128, 255, 256, 299):
            for k in ("conv1_state", "conv2_state", "conv2_out", "gru1", "gru2", "gru3", "gains"):
                assert np.array_equal(bits(a.debug(k, s)), bits(c.debug(k, s))), ("k_net without conv1", k, s, f)
                assert np.array_equal(bits(a.debug(k, s)), bits(b.debug(k, s))), ("k_net", k, s, f)
        assert np.array_equal(bits(oa), bits(oc)) and np.array_equal(bits(va), bits(vc)), f
        assert np.array_equal(bits(oa), bits(ob)) and np.array_equal(bits(va), bits(vb)), f
    a.destroy(); b.destroy(); c.destroy(); d.destroy()
    # pitch: group kernel (default: 16 streams per CTA, home + chain warps) vs the round-1 kernel (4 streams per CTA);
    # S = 300 leaves a partial group (12 of 16 streams) in the last CTA
    os.environ["RNNOISE_B200_PITCH_KERNEL"] = "v1"
    a = rb.Batch(model, S)
    os.environ["RNNOISE_B200_PITCH_KERNEL"] = "v2"
    b = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_PITCH_KERNEL"]
    for f in range(3 * frames):
        x = pcm[f % frames]
        oa, va = a.process(x); ob, vb = b.process(x)
        assert np.array_equal(bits(oa), bits(ob)) and np.array_equal(bits(va), bits(vb)), f
        for s in (0, 15, 16, 143, 287, 288, 299):
            for k in ("pitch", "features", "P"):
                assert np.array_equal(bits(a.debug(k, s)), bits(b.debug(k, s))), (k, s, f)
    a.destroy(); b.destroy()
    model.free()


def test_async_pipelined_host_call_equals_synchronous(rb, models_dir):
    """rnnoise_process_frame_batch_async (3-stream, double-buffered H2D / compute / D2H pipeline) must
    deliver exactly what the synchronous host call delivers, frame after frame."""
    import torch
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 500, 9
    a, b = rb.Batch(model, S), rb.Batch(model, S)
    pcm = torch.from_numpy(batch_pcm(S, frames)).pin_memory()
    outs = [torch.empty(S, 480).pin_memory() for _ in range(frames)]
    vads = [torch.empty(S).pin_memory() for _ in range(frames)]
    for f in range(frames):
        b.process_ptr_async(outs[f].data_ptr(), pcm[f].data_ptr(), vads[f].data_ptr())
    b.sync()
    for f in range(frames):
        ro, rv = a.process(pcm[f].numpy())
        assert np.array_equal(bits(outs[f].numpy()), bits(ro)) and np.array_equal(bits(vads[f].numpy()), bits(rv)), f
    a.destroy(); b.destroy(); model.free()


def test_prefilter_hint_path_equals_plain_device_call(rb, models_dir):
    """rnnoise_batch_prefilter_device() only moves the high-pass biquad of the next frame onto another
    stream; results must not change."""
    import torch
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 200, 8
    a, b = rb.Batch(model, S), rb.Batch(model, S)
    pcm = torch.from_numpy(batch_pcm(S, frames)).cuda()
    oa, ob = torch.empty(S, 480, device="cuda"), torch.empty(S, 480, device="cuda")
    va, vb = torch.empty(S, device="cuda"), torch.empty(S, device="cuda")
    torch.cuda.synchronize()
    b.prefilter_device(pcm[0].data_ptr())
    for f in range(frames):
        a.process_device(oa.data_ptr(), pcm[f].data_ptr(), va.data_ptr())
        if f + 1 < frames:
            b.prefilter_device(pcm[f + 1].data_ptr())
        b.process_device(ob.data_ptr(), pcm[f].data_ptr(), vb.data_ptr())
        a.sync(); b.sync()
        assert torch.equal(oa, ob) and torch.equal(va, vb), f
    a.destroy(); b.destroy(); model.free()


def test_two_stream_overlap_is_race_free(rb, models_dir):
    """The analysis of frame f+1 overlaps network + synthesis of frame f on another stream (triple-
    buffered spectra, double-buffered features).  A long back-to-back run through the pipelined call
    must equal the same run with RNNOISE_B200_OVERLAP=0 bit for bit."""
    import torch
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 1500, 40
    os.environ["RNNOISE_B200_OVERLAP"] = "0"
    a = rb.Batch(model, S)
    del os.environ["RNNOISE_B200_OVERLAP"]
    b = rb.Batch(model, S)
    pcm = torch.from_numpy(batch_pcm(S, frames)).pin_memory()
    oa = [torch.empty(S, 480).pin_memory() for _ in range(frames)]
    ob = [torch.empty(S, 480).pin_memory() for _ in range(frames)]
    va = [torch.empty(S).pin_memory() for _ in range(frames)]
    vb = [torch.empty(S).pin_memory() for _ in range(frames)]
    for f in range(frames):
        a.process_ptr_async(oa[f].data_ptr(), pcm[f].data_ptr(), va[f].data_ptr())
        b.process_ptr_async(ob[f].data_ptr(), pcm[f].data_ptr(), vb[f].data_ptr())
    a.sync(); b.sync()
    for f in range(frames):
        assert torch.equal(oa[f], ob[f]) and torch.equal(va[f], vb[f]), f
    a.destroy(); b.destroy(); model.free()


def test_int16_pcm_io_matches_demo_semantics(rb, models_dir):
    """rnnoise_process_frame_batch_s16: int16 in (widened exactly) / int16 out (C cast of the float result,
    examples/rnnoise_demo.c:56-58) must equal the float API followed by that cast."""
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, frames = 130, 12
    a, b = rb.Batch(model, S), rb.Batch(model, S)
    pcm = batch_pcm(S, frames)                     # integer-valued floats in int16 range
    for f in range(frames):
        of, vf = a.process(pcm[f])
        o16, v16 = b.process_s16(pcm[f].astype(np.int16))
        assert np.array_equal(o16, of.astype(np.int32).astype(np.int16)) and np.array_equal(bits(vf), bits(v16)), f
    a.destroy(); b.destroy(); model.free()


@pytest.mark.parametrize("chunk", [None, "5"])
def test_multi_frame_calls_equal_frame_at_a_time(rb, models_dir, chunk, monkeypatch):
    """rnnoise_process_frames_batch{,_s16,_device}: T frames per call over [S][T*480] buffers are
    bit-identical to T single-frame calls, across chunk boundaries (T not a multiple of the staging
    chunk), across consecutive multi-frame calls, and when mixed with single-frame calls."""
    import torch
    if chunk:
        monkeypatch.setenv("RNNOISE_B200_MULTI_CHUNK", chunk)
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    S, T1, T2 = 70, 23, 9
    frames = T1 + 1 + T2
    a, b, c, d = (rb.Batch(model, S) for _ in range(4))
    pcm = batch_pcm(S, frames)                     # [frames][S][480], integer-valued
    ref_out = np.empty((S, frames * 480), np.float32); ref_vad = np.empty((S, frames), np.float32)
    for f in range(frames):
        o, v = a.process(pcm[f])
        ref_out[:, f * 480:(f + 1) * 480] = o; ref_vad[:, f] = v
    by_stream = np.ascontiguousarray(pcm.transpose(1, 0, 2).reshape(S, frames * 480))
    # host float: T1 frames, one single-frame call, T2 frames
    o1, v1 = b.process_frames(by_stream[:, :T1 * 480])
    om, vm = b.process(pcm[T1])
    o2, v2 = b.process_frames(by_stream[:, (T1 + 1) * 480:])
    got = np.concatenate([o1, om, o2], axis=1); gv = np.concatenate([v1, vm[:, None], v2], axis=1)
    assert np.array_equal(bits(got), bits(ref_out)) and np.array_equal(bits(gv), bits(ref_vad))
    # host int16, whole signal in one call
    o16, v16 = c.process_frames(by_stream.astype(np.int16))
    assert o16.dtype == np.int16 and np.array_equal(o16, ref_out.astype(np.int32).astype(np.int16))
    assert np.array_equal(bits(v16), bits(ref_vad))
    # device pointers, in place
    dbuf = torch.from_numpy(by_stream).cuda(); dv = torch.empty(S, frames, device="cuda")
    torch.cuda.synchronize()
    d.process_frames_device(dbuf.data_ptr(), dbuf.data_ptr(), dv.data_ptr(), frames)
    d.sync()
    assert np.array_equal(bits(dbuf.cpu().numpy()), bits(ref_out)) and np.array_equal(bits(dv.cpu().numpy()), bits(ref_vad))
    for x in (a, b, c, d):
        x.destroy()
    model.free()


def test_train_features_match_training_reference_goldens(rb, models_dir):
    """rnnoise_batch_train_features: records bit-identical to the unmodified reference built with
    -DTRAINING=1 running the dump_features frame loop (tests/golden/ref_train.npz, made by
    tests/golden/make_golden_train.py); host and device entry points agree."""
    import torch
    from rnnoise_b200.synth_pcm import train_pair, train_params
    g = np.load(os.path.join(GOLD, "ref_train.npz"))
    streams, frames = [int(s) for s in g["streams"]], int(g["frames"])
    S = len(streams)
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    a, b = rb.Batch(model, S), rb.Batch(model, S)
    pairs = [train_pair(s, frames) for s in streams]
    par = [train_params(s) for s in streams]
    lowpass = np.array([p[0] for p in par], np.int32); band_lp = np.array([p[1] for p in par], np.int32)
    noise_free = np.array([p[2] for p in par], np.int32)
    dl, db, dn = (torch.from_numpy(x).cuda() for x in (lowpass, band_lp, noise_free))
    for f in range(frames):
        clean = np.stack([p[0][f] for p in pairs]); noisy = np.stack([p[1][f] for p in pairs])
        vad = np.array([float((f // 7 + s) % 2) for s in streams], np.float32)
        rec = a.train_features(clean, noisy, vad, noise_free, lowpass, band_lp)
        assert np.array_equal(bits(rec), bits(g["rec"][f])), (f, np.argwhere(bits(rec) != bits(g["rec"][f]))[:5])
        assert np.array_equal(np.array([int(a.debug("silence", i)[0]) for i in range(S)]), g["quiet"][f]), f
        dc, dno, dv = (torch.from_numpy(x).cuda() for x in (clean, noisy, vad))
        drec = torch.empty(S, 98, device="cuda")
        torch.cuda.synchronize()
        assert rb.lib().rnnoise_batch_train_features_device(b.handle, drec.data_ptr(), dc.data_ptr(), dno.data_ptr(), dv.data_ptr(),
                                                            dn.data_ptr(), dl.data_ptr(), db.data_ptr()) == 0
        b.sync()
        assert np.array_equal(bits(drec.cpu().numpy()), bits(rec)), f
    # defaults (all optional arrays NULL): no low-pass, vad target 0, noise present
    c = rb.Batch(model, S)
    r0 = c.train_features(np.stack([p[0][0] for p in pairs]), np.stack([p[1][0] for p in pairs]))
    assert r0.shape == (S, 98) and np.all(r0[:, 97] == 0)
    for x in (a, b, c):
        x.destroy()
    model.free()


@pytest.mark.parametrize("S,lanes,expect", [(300, "2", 2), (600, "4", 3)])
def test_lanes_do_not_change_results(rb, models_dir, S, lanes, expect, monkeypatch):
    """A batch split into lanes (sub-batches on their own CUDA streams) must be indistinguishable from a
    single-lane batch: host float / int16 / multi-frame calls, the device-pointer call on a caller stream,
    per-stream reset and debug reads (routed to the owning lane).  Lanes are whole 128-stream tiles except
    the last: 300 streams -> 256 + 44; 600 streams asked for 4 lanes -> 256 + 256 + 88 (three lanes)."""
    import torch
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    frames = 8
    monkeypatch.setenv("RNNOISE_B200_LANES", "1")
    ref, ref16 = rb.Batch(model, S), rb.Batch(model, S)
    monkeypatch.setenv("RNNOISE_B200_LANES", lanes)
    a, a16, dev, multi = (rb.Batch(model, S) for _ in range(4))
    assert ref.lanes == 1 and a.lanes == expect
    pcm = batch_pcm(S, frames)
    st = torch.cuda.Stream()
    dev.set_stream(st.cuda_stream)
    outs = []
    for f in range(frames):
        if f == 4:
            for b in (ref, a, dev):
                b.reset_stream(7); b.reset_stream(S - 1)
        ro, rv = ref.process(pcm[f]); outs.append((ro, rv))
        o, v = a.process(pcm[f])
        assert np.array_equal(bits(o), bits(ro)) and np.array_equal(bits(v), bits(rv)), f
        for s in (0, 127, 128, 255, 256, S - 1):
            for k in ("features", "gains", "gru3"):
                assert np.array_equal(bits(a.debug(k, s)), bits(ref.debug(k, s))), (k, s, f)
        r16, rv16 = ref16.process_s16(pcm[f].astype(np.int16)); o16, v16 = a16.process_s16(pcm[f].astype(np.int16))
        assert np.array_equal(r16, o16) and np.array_equal(bits(rv16), bits(v16)), f
        with torch.cuda.stream(st):
            d = torch.from_numpy(pcm[f]).cuda(non_blocking=False); dv = torch.empty(S, device="cuda")
            dev.process_device(d.data_ptr(), d.data_ptr(), dv.data_ptr())
            got, gotv = d.cpu().numpy(), dv.cpu().numpy()     # ordered on the caller's stream only
        assert np.array_equal(bits(got), bits(ro)) and np.array_equal(bits(gotv), bits(rv)), f
    # multi-frame call over the first 4 frames (before the resets)
    by_stream = np.ascontiguousarray(pcm[:4].transpose(1, 0, 2).reshape(S, 4 * 480))
    mo, mv = multi.process_frames(by_stream)
    want = np.concatenate([outs[f][0] for f in range(4)], axis=1); wantv = np.stack([outs[f][1] for f in range(4)], axis=1)
    assert np.array_equal(bits(mo), bits(want)) and np.array_equal(bits(mv), bits(wantv))
    for b in (ref, ref16, a, a16, dev, multi):
        b.destroy()
    model.free()


def test_edge_case_signals_and_poisoned_neighbours(rb, port_default, models_dir):
    """Full-scale square wave, impulses, DC, vanishing (incl. denormal) noise, clipped noise and gaps of digital silence as
    streams of one batch: every DSP quantity, the PCM and the VAD stay bit-identical to the port.  Two more streams carry
    one NaN / one Inf sample (the reference's state is poisoned for good by either): their NaNs must not reach any other
    stream of the batch -- the ordinary stream next to them stays bit-exact."""
    from test_dsp_emulation import _edge_signals
    frames = 40
    sigs = list(_edge_signals(frames))
    names = [n for n, _ in sigs] + ["ordinary"]
    pcm = np.stack([x.reshape(frames, 480) for _, x in sigs] + [stream_pcm(3, frames)], axis=1)   # [frames][S][480]
    S = pcm.shape[1]
    finite = [bool(np.isfinite(pcm[:, i]).all()) for i in range(S)]
    model = rb.Model(os.path.join(models_dir, "default.bin"))
    batch = rb.Batch(model, S)
    states = [port_default.create() for _ in range(S)]
    nan_pos_mismatch = 0
    for f in range(frames):
        out, vad = batch.process(pcm[f])
        for i in range(S):
            r = port_default.process_frame(states[i], pcm[f, i])
            tag = f"frame {f} stream {names[i]}"
            if finite[i]:
                assert int(batch.debug("silence", i)[0]) == r["silence"] and int(batch.debug("pitch", i)[0]) == r["pitch"], tag
                for key in ("xb", "X", "P", "Ex", "Ep", "Exp", "features"):
                    assert np.array_equal(bits(batch.debug(key, i)), bits(r[key])), f"{key} not bit-exact, {tag}"
                assert np.array_equal(bits(out[i]), bits(r["out"])), f"pcm, {tag}"
                assert np.array_equal(bits(vad[i:i + 1]), bits(np.float32([r["vad"]]))), f"vad, {tag}"
            else:
                nan_pos_mismatch += int((np.isnan(out[i]) != np.isnan(r["out"])).sum())
    print("NaN-position differences on the poisoned streams (informative):", nan_pos_mismatch)
    for st in states:
        port_default.destroy(st)
    batch.destroy()
    model.free()
