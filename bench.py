#!/usr/bin/env python3
"""bench.py -- 10 ms frames/sec of the batched denoise hot path (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--streams S] [--impl b200|reference] [--dump-outputs DIR]
  (N > 1: launched by torchrun, one rank per GPU; streams shard with no collective -> "weak")

One "step" = one call of the hot path = one 480-sample frame for each of S streams resident on a
GPU (default S = 4096 = BASELINE configs[1], default synthetic model).  Prints ONE JSON line:
  value      whole-job frames/s, PCM already resident in HBM (rnnoise_process_frame_batch_device)
  e2e        same metric through the host-buffer C-ABI call rnnoise_process_frame_batch():
             pinned host in -> H2D -> kernels -> D2H -> pinned host out, all inside the timed region
  roofline   dominant kernel: algorithmic bytes / CUDA-event duration vs MEASURED_PEAKS.json
  cpu_baseline  the unmodified reference (oracle/_ref, AVX2 RTCD build) on this box's host cores
--impl reference times that CPU reference arm alone on the same workload.
--dump-outputs DIR writes what the last timed step computed (denoised PCM and VAD of every stream, see dump_outputs)
so that two builds can be compared output for output: the inputs depend only on the arguments.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

FRAME = 480
POOL_FRAMES = 32          # distinct frames per pooled stream (device-resident input rotates through them)
POOL_STREAMS = 128        # distinct synthetic streams, tiled over S
MODEL = os.path.join(ROOT, "tests", "golden", "models", "default.bin")
# Algorithmic HBM bytes per stream-frame (DESIGN.md "Kernels"): whole pipeline 43 344 (SURVEY 8d);
# per kernel, counting each array the kernel must read or write once:
KERNEL_BYTES = {
    "k_biquad": 480 * 4 * 2 + 16,                                   # in -> xb, hp state
    "k_pitch": (480 + 1248 + 480 + 4) * 4,                          # xb, ring history read, new frame appended, pitch state
    "k_spectrum": (1728 + 2 * 962 + 96 + 65 + 1 + 2) * 4,           # ring (both windows), X+P, bands, features, flags
    "k_synthesis": (2 * 962 + 96 + 32 + 32 + 2 * 32 + 2 * 480 + 480) * 4,
    # conv1 (features, conv1 memory r/w, conv2 operand row r/w) + conv2 + 3 GRU layers (fp32 state r/w, u8 mirrors), default dims
    "k_net": 1292 + 2688 + 3 * 6144,
    "k_heads": 6276,
}


DUMP_LIMIT = 64 << 20   # bytes written by --dump-outputs at most


def dump_outputs(d, out, vad):
    """out [S][480], vad [S] (float32) of the last timed step -> d/pcm.npy, d/vad.npy.  Past DUMP_LIMIT bytes a fixed,
    seeded sample of the streams is written instead, their indices in d/stream_index.npy."""
    os.makedirs(d, exist_ok=True)
    S = out.shape[0]
    # per kept stream: 480 PCM + 1 VAD float32 + the float64 index; 4 KB for the three .npy headers
    keep = (DUMP_LIMIT - 4096) // ((FRAME + 1) * 4 + 8)
    if S > keep:
        idx = np.sort(np.random.default_rng(0).choice(S, keep, replace=False))
        out, vad = out[idx], vad[idx]
        np.save(os.path.join(d, "stream_index.npy"), idx.astype(np.float64))
    np.save(os.path.join(d, "pcm.npy"), np.ascontiguousarray(out, np.float32))
    np.save(os.path.join(d, "vad.npy"), np.ascontiguousarray(vad, np.float32))


def world():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def pool_frames(S):
    """Frames in the rotating input pool: 32, fewer for very large S (keeps pinned memory <= ~1 GB)."""
    return int(max(4, min(POOL_FRAMES, (1 << 30) // (S * FRAME * 4))))


def base_pool(S):
    """float32 [pool_frames(S)][min(POOL_STREAMS, S)][480]: the distinct synthetic streams of the input pool."""
    from rnnoise_b200.synth_pcm import batch_pcm
    return batch_pcm(min(POOL_STREAMS, S), pool_frames(S))


def make_pool(S):
    """float32 [pool_frames(S)][S][480]: POOL_STREAMS distinct synthetic streams tiled to S (stream s = pool stream s % 128)."""
    base = base_pool(S)
    reps = (S + base.shape[1] - 1) // base.shape[1]
    return np.ascontiguousarray(np.tile(base, (1, reps, 1))[:, :S])


class ClockSampler(threading.Thread):
    """Samples SM clock + throttle reasons during the timed region (NVML)."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.samples, self.reasons, self.max_mhz, self._stop = [], set(), None, threading.Event()
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def run(self):
        if not self.nv:
            return
        names = {"hw_slowdown": 0x8, "sw_power_cap": 0x4, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20,
                 "hw_power_brake_slowdown": 0x80}
        while not self._stop.is_set():
            try:
                self.samples.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
                try:
                    r = self.nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    r = self.nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for n, bit in names.items():
                    if r & bit:
                        self.reasons.add(n)
            except Exception:
                pass
            time.sleep(0.02)

    def stop(self):
        self._stop.set()
        med = float(np.median(self.samples)) if self.samples else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(self.samples)}


REF_REPEATS = 5     # BASELINE.md section 3: repeat the CPU measurement >= 5 times, report median and best


def has_vnni():
    try:
        return any(l.startswith("flags") and " avx_vnni" in l for l in open("/proc/cpuinfo"))
    except Exception:
        return False


_pool_file = {}


def pool_file(S):
    """The GPU arm's input pool written once for the CPU arm (same PCM on both sides): [frames][streams][480] float32."""
    if S not in _pool_file:
        base = base_pool(S)
        d = "/dev/shm" if os.path.isdir("/dev/shm") else "/tmp"
        path = os.path.join(d, f"rnnoise_b200_pool_{os.getpid()}_{S}.f32")
        base.astype(np.float32).tofile(path)
        import atexit
        atexit.register(lambda: os.path.exists(path) and os.remove(path))
        _pool_file[S] = (path, base.shape[1], base.shape[0])
    return _pool_file[S]


def run_reference(S, steps, warmup, threads=None, repeats=1, vnni=False, model=None, pool_S=None):
    """Times the unmodified reference (oracle/_ref) on the host cores; returns dict or None."""
    from oracle import refbind
    from rnnoise_b200 import weights
    d = weights.describe(open(model or MODEL, "rb").read())    # the reference's model dims are compile-time: one build per (cond, gru)
    exe = refbind.bench_path(d["cond"], d["gru"], vnni=vnni)
    if not os.path.exists(exe):
        return None
    threads = threads or len(os.sched_getaffinity(0))
    cmd = [exe, model or MODEL, str(S), str(steps), str(warmup), str(threads), str(repeats)]
    if pool_S:
        path, ps, pf = pool_file(pool_S)
        cmd += [path, str(ps), str(pf)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    if r.returncode != 0:
        return None
    d = json.loads(r.stdout.strip().splitlines()[-1])
    d["threads"] = min(threads, S)
    return d


def best_reference_threads(S, model=None):
    """Quick sweep: containers often expose more logical CPUs than their CPU quota; pick the thread
    count that gives the reference its best throughput on this box."""
    n = len(os.sched_getaffinity(0))
    best, best_t = None, n
    for t in sorted({n, max(1, n // 2), max(1, n // 4), max(1, n // 8)}, reverse=True):
        r = run_reference(min(S, 8 * t), 12, 3, threads=t, model=model)
        if r and (best is None or r["frames_per_s"] > best):
            best, best_t = r["frames_per_s"], t
    return best_t, best


def reference_baseline(S, budget_s, model=None, warmup=5):
    """BASELINE.md section 3 protocol: the unmodified reference (RTCD/AVX2 build), the thread count that is best
    on this box, the SAME PCM pool as the GPU arm, REF_REPEATS back-to-back repeats -> median (the value) and
    best; plus the AVX-VNNI build of the same sources when the host has the instruction.  `budget_s` bounds the
    CPU work of the main run."""
    threads, rate = best_reference_threads(S, model)
    if not rate:
        return None
    steps = int(max(3, min(400, budget_s / REF_REPEATS * rate / S)))
    ref = run_reference(S, steps, warmup, threads=threads, repeats=REF_REPEATS, model=model, pool_S=S)
    if ref is None:
        return None
    ref["steps_per_repeat"] = steps
    if has_vnni():
        v = run_reference(S, steps, warmup, threads=threads, repeats=3, vnni=True, model=model, pool_S=S)
        if v:
            ref["vnni"] = {"value": v["frames_per_s"], "best": v["best_frames_per_s"], "build": "same sources, nnet_avx2.c with -mavxvnni (vec_avx.h:623 branch)"}
    return ref


def cpu_baseline_dict(ref, S):
    return {"value": ref["frames_per_s"], "best": ref["best_frames_per_s"], "repeats": ref["repeat_frames_per_s"], "unit": "frames/s",
            "cores": ref["threads"], "kind": "reference", "vnni": ref.get("vnni"),
            "sample": f"{S} streams x {ref['steps_per_repeat']} frames x {REF_REPEATS} repeats (value = median, best beside it), same PCM pool as the "
                      f"GPU arm, unmodified xiph/rnnoise RTCD/AVX2 build via oracle/_ref, {ref['threads']} threads (best of a thread sweep "
                      f"over the {len(os.sched_getaffinity(0))} logical CPUs the container exposes), {cpu_model()}"}


def cpu_model():
    try:
        for l in open("/proc/cpuinfo"):
            if l.startswith("model name"):
                return l.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def single_process(a, cfg, S, K, Wm):
    """One host thread, G GPUs: rnnoise_batch_create_multi shards G * S streams contiguously over the devices; the
    device-resident arm times every device with its own CUDA events (value = all streams / max over devices), the
    e2e arm goes through the ordinary host-buffer call on one [G * S][480] pinned buffer."""
    import torch
    import rnnoise_b200
    G = a.gpus
    model = rnnoise_b200.Model(MODEL)
    batch = rnnoise_b200.Batch(model, G * S, devices=list(range(G)))
    assert batch.nb_devices == G and all(batch.shard(k) == (k, k * S, S) for k in range(G))
    base = torch.from_numpy(make_pool(S))
    F = base.shape[0]
    pool_d = [base.to(f"cuda:{k}") for k in range(G)]
    out_d = [torch.empty(S, FRAME, device=f"cuda:{k}") for k in range(G)]
    vad_d = [torch.empty(S, device=f"cuda:{k}") for k in range(G)]
    streams = [torch.cuda.Stream(torch.device("cuda", k)) for k in range(G)]
    batch.set_stream_multi([s.cuda_stream for s in streams])

    def step(i):
        batch.prefilter_device_multi([p[(i + 1) % F].data_ptr() for p in pool_d])
        batch.process_device_multi([o.data_ptr() for o in out_d], [p[i % F].data_ptr() for p in pool_d], [v.data_ptr() for v in vad_d])

    def sync_all():
        for k in range(G):
            torch.cuda.synchronize(k)

    batch.prefilter_device_multi([p[0].data_ptr() for p in pool_d])
    for i in range(Wm):
        step(i)
    sync_all()
    sampler = ClockSampler(0)
    sampler.start()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(G)]
    t0 = time.perf_counter()
    for k in range(G):
        with torch.cuda.device(k):
            ev[k][0].record(streams[k])
    for i in range(K):
        step(Wm + i)
    for k in range(G):
        with torch.cuda.device(k):
            ev[k][1].record(streams[k])
    sync_all()
    wall_ms = (time.perf_counter() - t0) * 1e3
    ms = max(e0.elapsed_time(e1) for e0, e1 in ev)
    clocks = sampler.stop()
    if a.dump_outputs:
        dump_outputs(a.dump_outputs, torch.cat([o.cpu() for o in out_d]).numpy(), torch.cat([v.cpu() for v in vad_d]).numpy())
    batch.process_device_multi([o.data_ptr() for o in out_d], [p[(Wm + K) % F].data_ptr() for p in pool_d], [v.data_ptr() for v in vad_d])
    batch.sync()
    value = G * S * K / (ms * 1e-3)
    # e2e: one [G * S][480] pinned buffer per pool frame, host-buffer call of the whole batch
    Fh = min(F, max(2, (1 << 30) // (G * S * FRAME * 4)))
    pool_h = torch.cat([base[:Fh]] * G, dim=1).contiguous().pin_memory()
    NBUF = 4
    out_h = [torch.empty(G * S, FRAME).pin_memory() for _ in range(NBUF)]
    vad_h = [torch.empty(G * S).pin_memory() for _ in range(NBUF)]
    for i in range(4):
        batch.process_ptr_async(out_h[i % NBUF].data_ptr(), pool_h[i % Fh].data_ptr(), vad_h[i % NBUF].data_ptr())
    batch.sync()
    t0 = time.perf_counter()
    for i in range(K):
        batch.process_ptr_async(out_h[i % NBUF].data_ptr(), pool_h[i % Fh].data_ptr(), vad_h[i % NBUF].data_ptr())
    batch.sync()
    ms_e = (time.perf_counter() - t0) * 1e3
    line = {"metric": "10ms frames/sec", "value": value, "unit": "frames/s", "n_gpus": G, "steps": K, "warmup": Wm, "ms_per_step": ms / K,
            "wall_ms_per_step": wall_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "int8 (u8 x s8 -> s32) + fp32", "data": "synthetic", "config": dict(cfg, streams_total=G * S),
            "launch": "single process: one host thread drives all GPUs through rnnoise_batch_create_multi (no torchrun, no NCCL)",
            "realtime_streams_per_gpu": value / G / 100.0, "clocks": clocks, "lanes": batch.lanes,
            "e2e": {"value": G * S * K / (ms_e * 1e-3), "unit": "frames/s", "steps": K, "ms_per_step": ms_e / K,
                    "h2d_bytes_per_step": G * S * FRAME * 4, "d2h_bytes_per_step": G * S * FRAME * 4 + G * S * 4,
                    "api": "rnnoise_process_frame_batch_async on a multi-device batch + rnnoise_batch_sync"},
            "gpu_launches": K * batch.launches_per_frame}
    print(json.dumps(line))
    batch.destroy()
    model.free()


def main():
    global POOL_FRAMES
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=2000)   # ~0.7 s timed region at 4096 streams: enough clock samples
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--streams", type=int, default=4096, help="streams per GPU")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--model", default="default", help="model name under tests/golden/models (default, little, ...) or a blob path")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the outputs of the last timed step to DIR/<name>.npy")
    ap.add_argument("--single-process", action="store_true",
                    help="with --gpus N and no torchrun: ONE process drives N GPUs through rnnoise_batch_create_multi (C ABI sharding)")
    a = ap.parse_args()
    global MODEL
    if a.model != "default":
        MODEL = a.model if os.path.exists(a.model) else os.path.join(ROOT, "tests", "golden", "models", a.model + ".bin")
    W, rank, local = world()
    S, K, Wm = a.streams, a.steps, max(a.warmup, 3)
    cfg = {"workload": f"{S} concurrent 48 kHz mono streams per GPU, {a.model} synthetic model (int8 block-sparse GRUs), "
                       f"one 480-sample frame per stream per step", "streams_per_gpu": S, "frame": FRAME,
           "model": os.path.relpath(MODEL, ROOT),
           "l2": f"per-step state+I/O working set {S * 43344 / 1e6:.0f} MB vs 50 MB L2; input rotates through a "
                 f"{pool_frames(S)}-frame device pool ({pool_frames(S) * S * FRAME * 4 / 1e6:.0f} MB)"}

    if a.impl == "reference":
        # CPU arm: rank 0 alone runs it; other ranks exit quietly.
        if rank != 0:
            return
        total_S = S * max(a.gpus, 1)
        # every step = one frame of all streams on the host cores; the sample is bounded to about a minute of
        # CPU work in total (the rate does not depend on how many frames are run)
        ref = reference_baseline(total_S, 60.0, model=MODEL, warmup=min(Wm, 5))
        if ref is None:
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/ref_bench not built (needs the reference sources at build time)"}))
            return
        v = ref["frames_per_s"]
        print(json.dumps({"impl": "reference", "metric": "10ms frames/sec", "value": v, "unit": "frames/s", "n_gpus": a.gpus,
                          "steps": K, "warmup": Wm, "ms_per_step": 1e3 * ref["elapsed_s"] / ref["steps_per_repeat"], "higher_is_better": True,
                          "scaling": "weak", "vs_baseline": None, "dtype": "int8+fp32 (AVX2)", "data": "synthetic",
                          "config": dict(cfg, streams_total=total_S),
                          "cpu_baseline": cpu_baseline_dict(ref, total_S),
                          "e2e": {"value": v, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return

    import torch
    import rnnoise_b200
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (no CPU fallback)")
    if a.single_process and W == 1 and a.gpus > 1:
        return single_process(a, cfg, S, K, Wm)
    if W > 1:
        import torch.distributed as dist
        # NCCL's log (version banner, INFO lines when the caller sets NCCL_DEBUG=INFO to check the ranks) goes to
        # stderr, so that stdout carries the one JSON line only; NCCL_DEBUG itself is left to the caller
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if not os.path.exists(rnnoise_b200.LIB_PATH):
        from rnnoise_b200 import build
        build.build()
    model = rnnoise_b200.Model(MODEL)
    batch = rnnoise_b200.Batch(model, S, local)
    pool_h = torch.from_numpy(make_pool(S)).pin_memory()           # [POOL][S][480] pinned host
    POOL_FRAMES = pool_h.shape[0]
    pool_d = pool_h.to(dev)                                        # device-resident inputs
    out_d = torch.empty(S, FRAME, device=dev)
    vad_d = torch.empty(S, device=dev)
    # a dedicated non-default stream: handle 0 (the legacy default stream) means "private stream" to
    # rnnoise_batch_set_stream(), and events must be recorded on the stream the kernels run on.
    stream = torch.cuda.Stream(dev, priority=int(os.environ.get("BENCH_STREAM_PRIORITY", "-1")))
    torch.cuda.set_stream(stream)
    assert stream.cuda_stream != 0
    batch.set_stream(stream.cuda_stream)

    def step_device(i):
        # the input pool is device-resident, so the next frame's high-pass prefilter can be hinted ahead
        batch.prefilter_device(pool_d[(i + 1) % POOL_FRAMES].data_ptr())
        batch.process_device(out_d.data_ptr(), pool_d[i % POOL_FRAMES].data_ptr(), vad_d.data_ptr())

    def barrier():
        if W > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    # ---- device-resident throughput (value) ----
    batch.prefilter_device(pool_d[0].data_ptr())
    for i in range(Wm):
        step_device(i)
    barrier()
    sampler = ClockSampler(local)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_wall = time.perf_counter()
    e0.record(stream)
    for i in range(K):
        step_device(Wm + i)
    e1.record(stream)
    barrier()
    wall_ms = (time.perf_counter() - t_wall) * 1e3
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    if a.dump_outputs:
        # the whole job's output: with several ranks every shard is gathered (rank r holds streams r*S .. r*S + S - 1)
        outs, vads = [out_d], [vad_d]
        if W > 1:
            outs, vads = [torch.empty_like(out_d) for _ in range(W)], [torch.empty_like(vad_d) for _ in range(W)]
            dist.all_gather(outs, out_d)
            dist.all_gather(vads, vad_d)
        if rank == 0:
            dump_outputs(a.dump_outputs, torch.cat(outs).cpu().numpy(), torch.cat(vads).cpu().numpy())
    # one prefilter hint is still pending (frame Wm+K): consume it so the host-call path starts clean
    batch.process_device(out_d.data_ptr(), pool_d[(Wm + K) % POOL_FRAMES].data_ptr(), vad_d.data_ptr())
    batch.sync()
    # the device-event time must explain the wall clock of the same region (guards against timing
    # the wrong stream): allow launch/sync slack only
    assert ms > 0.7 * wall_ms - 2.0, f"event time {ms:.2f} ms does not cover wall time {wall_ms:.2f} ms"
    if W > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    value = W * S * K / (ms * 1e-3)

    # ---- end-to-end through the host-buffer C-ABI call (e2e) ----
    # rnnoise_process_frame_batch_async(): every step copies that step's PCM from pinned host memory
    # to the device, runs the frame pipeline (10 kernels per lane) and copies PCM + VAD back to pinned host memory; consecutive
    # steps overlap on three streams.  Timed by wall clock around a fully synchronised region (covers
    # the last D2H), distinct output buffers per in-flight step.
    NBUF = 4
    out_h = [torch.empty(S, FRAME).pin_memory() for _ in range(NBUF)]
    vad_h = [torch.empty(S).pin_memory() for _ in range(NBUF)]
    Ke = K

    def step_host(i):
        batch.process_ptr_async(out_h[i % NBUF].data_ptr(), pool_h[i % POOL_FRAMES].data_ptr(), vad_h[i % NBUF].data_ptr())

    for i in range(4):
        step_host(i)
    batch.sync()
    barrier()
    t0 = time.perf_counter()
    for i in range(Ke):
        step_host(4 + i)
    batch.sync()
    ms_e = (time.perf_counter() - t0) * 1e3
    barrier()
    if W > 1:
        t = torch.tensor([ms_e], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_e = float(t.item())
    # also the plain synchronous call (one frame in flight), for reference
    t0 = time.perf_counter()
    for i in range(20):
        batch.process_ptr(out_h[0].data_ptr(), pool_h[i % POOL_FRAMES].data_ptr(), vad_h[0].data_ptr())
    ms_sync = (time.perf_counter() - t0) * 1e3 / 20
    # same pipeline with 16-bit PCM in both directions (rnnoise_process_frame_batch_s16_async)
    in16 = pool_h[:min(8, POOL_FRAMES)].to(torch.int16).pin_memory()
    out16 = [torch.empty(S, FRAME, dtype=torch.int16).pin_memory() for _ in range(NBUF)]
    for i in range(4):
        batch.process_ptr_s16_async(out16[i % NBUF].data_ptr(), in16[i % in16.shape[0]].data_ptr(), vad_h[i % NBUF].data_ptr())
    batch.sync()
    t0 = time.perf_counter()
    for i in range(Ke):
        batch.process_ptr_s16_async(out16[i % NBUF].data_ptr(), in16[i % in16.shape[0]].data_ptr(), vad_h[i % NBUF].data_ptr())
    batch.sync()
    ms_16 = (time.perf_counter() - t0) * 1e3
    e2e = {"value": W * S * Ke / (ms_e * 1e-3), "unit": "frames/s", "steps": Ke, "ms_per_step": ms_e / Ke,
           "int16_pcm": {"value": S * Ke / (ms_16 * 1e-3), "h2d_bytes_per_step": S * FRAME * 2, "d2h_bytes_per_step": S * FRAME * 2 + S * 4,
                         "note": "this rank only"},
           "h2d_bytes_per_step": S * FRAME * 4, "d2h_bytes_per_step": S * FRAME * 4 + S * 4,
           "api": "rnnoise_process_frame_batch_async + rnnoise_batch_sync (pinned host buffers; H2D, kernels, D2H of every step inside the wall-clock region)",
           "synchronous_call_ms_per_step": ms_sync}

    # ---- per-kernel CUDA-event timing for the roofline (separate pass, same workload) ----
    batch.profile(True)
    Kp = max(5, min(K, 50))
    for i in range(Kp):
        batch.process_device(out_d.data_ptr(), pool_d[i % POOL_FRAMES].data_ptr(), vad_d.data_ptr())
    times, nprof = batch.profile_read()
    batch.profile(False)
    lanes = batch.lanes                                            # sub-batches run side by side (include/rnnoise.h)
    kernels = {k: v / nprof for k, v in times.items() if k != "-"}   # ms per step and kernel, summed over the lanes' launches
    top = max(kernels, key=kernels.get)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)
    top_bytes = KERNEL_BYTES.get(top, 43344) * S // lanes           # one launch covers one lane's streams
    ms_launch = kernels[top] / lanes
    achieved = top_bytes / (ms_launch * 1e-3) / 1e9
    roof = {"kernel": top, "bound": "hbm", "achieved": achieved, "peak": hbm, "unit": "GB/s", "frac": achieved / hbm,
            "peak_source": "MEASURED_PEAKS.json hbm_gbs (measured)" if "hbm_gbs" in peaks else "H100 SXM data sheet, 3350 GB/s",
            "algorithmic_bytes_per_launch": top_bytes, "ms_per_launch": ms_launch, "launches_per_step": lanes,
            "streams_per_launch": S // lanes,
            "kernel_ms_per_step": kernels, "kernel_share": {k: v / sum(kernels.values()) for k, v in kernels.items()},
            "pipeline": {"algorithmic_bytes_per_stream_frame": 43344,
                         "achieved_GBps": 43344 * S * K / (ms * 1e-3) / 1e9 / 1.0,
                         "frac": 43344 * S * K / (ms * 1e-3) / 1e9 / hbm}}

    if rank == 0:
        cpu = None
        if W == 1 and not a.no_cpu_baseline:
            try:
                ref = reference_baseline(S, 20.0, model=MODEL)
                cpu = cpu_baseline_dict(ref, S) if ref else None
            except Exception as ex:  # noqa: BLE001
                cpu = {"value": None, "unit": "frames/s", "cores": 0, "kind": "reference", "sample": f"failed: {ex}"}
        line = {"metric": "10ms frames/sec", "value": value, "unit": "frames/s", "n_gpus": W, "steps": K, "warmup": Wm,
                "ms_per_step": ms / K, "wall_ms_per_step": wall_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "int8 (u8 x s8 -> s32) + fp32", "data": "synthetic", "config": dict(cfg, streams_total=W * S),
                "realtime_streams_per_gpu": value / W / 100.0, "clocks": clocks, "e2e": e2e,
                "gpu_launches": K * batch.launches_per_frame, "lanes": lanes, "roofline": roof, "cpu_baseline": cpu}
        print(json.dumps(line))
    batch.destroy()
    model.free()
    if W > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
