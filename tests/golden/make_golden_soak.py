#!/usr/bin/env python3
"""Generates tests/golden/soak_<model>.npz, the reference side of tests/test_gpu_soak.py's soak comparison, from the
UNMODIFIED reference build (oracle/_ref, RTCD/AVX2 and generic-C builds; needs the reference sources at build time):

    python oracle/build_ref.py && python tests/golden/make_golden_soak.py

The soak runs 64 streams x 2000 frames of rnnoise_b200.synth_pcm.stream_pcm(stream, 2000).  A full copy of the
reference's PCM would be ~250 MB per model, so a fixed sample is stored:
  * PCM of both builds for STREAMS at FRAMES (frames spread over the whole run, the last one included),
  * VAD of both builds for STREAMS at every frame,
  * pitch period and silence flag of the RTCD build for the traced streams 0 .. TRACED-1 at every frame.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refbind import RefLib  # noqa: E402
from rnnoise_b200.synth_pcm import stream_pcm  # noqa: E402

T = 2000
STREAMS = (0, 15, 38, 63)                                  # 15: a stream with a 1 s digital-silence gap
FRAMES = np.unique(np.linspace(0, T - 1, 48).round().astype(np.int64))
TRACED = 8
HERE = os.path.dirname(os.path.abspath(__file__))


def run(lib, pcm, traced):
    st = lib.create()
    out = np.empty((T, 480), np.float32); vad = np.empty(T, np.float32)
    pitch = np.zeros(T, np.int16); sil = np.zeros(T, np.int8)
    for t in range(T):
        if traced:
            r = lib.process_frame_traced(st, pcm[t])
            out[t], vad[t], pitch[t], sil[t] = r["out"], r["vad"], r["pitch"], r["silence"]
        else:
            out[t], vad[t] = lib.process_frame(st, pcm[t])
    lib.destroy(st)
    return out, vad, pitch, sil


def main():
    for name in ("default", "hot", "little"):
        mp = os.path.join(HERE, "models", name + ".bin")
        avx, gen = RefLib(mp, "rtcd"), RefLib(mp, "generic")
        d = dict(frames_total=T, streams=np.array(STREAMS), frames=FRAMES, traced=TRACED)
        for s in sorted(set(STREAMS) | set(range(TRACED))):
            pcm = stream_pcm(s, T)
            a_out, a_vad, a_pitch, a_sil = run(avx, pcm, s < TRACED)
            if s < TRACED:
                d[f"s{s}_pitch"], d[f"s{s}_silence"] = a_pitch, a_sil
            if s in STREAMS:
                g_out, g_vad, _, _ = run(gen, pcm, False)
                d[f"s{s}_out"], d[f"s{s}_generic_out"] = a_out[FRAMES], g_out[FRAMES]
                d[f"s{s}_vad"], d[f"s{s}_generic_vad"] = a_vad, g_vad
        path = os.path.join(HERE, f"soak_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
