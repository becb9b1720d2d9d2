"""rnnoise_b200 -- host-side mirror of the C ABI in include/rnnoise.h (ctypes, no compute in Python).

The product is rnnoise_b200/librnnoise_b200.so (C host code + sm_90a CUDA kernels).  This module
only loads it and forwards calls with plain pointers, the way the reference's own callers
(examples/rnnoise_demo.c:40-66) use librnnoise.  It never falls back to a CPU path: importing works
without a GPU (so the ABI can be inspected), but creating a batch raises if the engine cannot come up.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# $RNNOISE_B200_LIB_PATH selects another build of the library (A/B measurements of two source states)
LIB_PATH = os.environ.get("RNNOISE_B200_LIB_PATH") or os.path.join(_HERE, "librnnoise_b200.so")
FRAME_SIZE = 480

# debug-read selectors (include/rnnoise.h)
DBG = dict(features=0, X=1, P=2, Ex=3, Ep=4, Exp=5, gains=6, lastg=7, xb=8, gru1=9, gru2=10, gru3=11,
           conv1_state=12, conv2_state=13, pitch=14, silence=15, conv2_out=16)

_lib = None


def shard(total_streams, world_size, rank):
    """Contiguous stream shard of `rank`: streams are independent, so multi-GPU use is one batch per
    device over [first, first + count) with no collective (SURVEY section 8e)."""
    base, rem = divmod(int(total_streams), int(world_size))
    first = rank * base + min(rank, rem)
    return first, base + (1 if rank < rem else 0)


def lib():
    """Loads the shared library (building is __graft_entry__.build()'s / build.py's job)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing -- run `python rnnoise_b200/build.py` (no CPU fallback exists)")
        L = C.CDLL(LIB_PATH)
        vp, ip, fp = C.c_void_p, C.c_int, C.POINTER(C.c_float)
        L.rnnoise_get_size.restype = ip
        L.rnnoise_get_frame_size.restype = ip
        L.rnnoise_model_from_filename.restype = vp; L.rnnoise_model_from_filename.argtypes = [C.c_char_p]
        L.rnnoise_model_from_buffer.restype = vp; L.rnnoise_model_from_buffer.argtypes = [vp, ip]
        L.rnnoise_model_free.argtypes = [vp]
        L.rnnoise_create.restype = vp; L.rnnoise_create.argtypes = [vp]
        L.rnnoise_destroy.argtypes = [vp]
        L.rnnoise_process_frame.restype = C.c_float; L.rnnoise_process_frame.argtypes = [vp, fp, fp]
        L.rnnoise_batch_create.restype = vp; L.rnnoise_batch_create.argtypes = [vp, ip, ip]
        L.rnnoise_batch_destroy.argtypes = [vp]
        L.rnnoise_batch_create_multi.restype = vp; L.rnnoise_batch_create_multi.argtypes = [vp, ip, C.POINTER(C.c_int), ip]
        L.rnnoise_batch_get_devices.restype = ip; L.rnnoise_batch_get_devices.argtypes = [vp]
        L.rnnoise_batch_get_shard.restype = ip; L.rnnoise_batch_get_shard.argtypes = [vp, ip] + [C.POINTER(C.c_int)] * 3
        L.rnnoise_process_frame_batch_device_multi.restype = ip
        L.rnnoise_process_frame_batch_device_multi.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
        L.rnnoise_batch_prefilter_device_multi.restype = ip; L.rnnoise_batch_prefilter_device_multi.argtypes = [vp, C.POINTER(vp)]
        L.rnnoise_batch_set_stream_multi.restype = ip; L.rnnoise_batch_set_stream_multi.argtypes = [vp, C.POINTER(vp)]
        L.rnnoise_batch_debug_set_frame_counter.restype = ip; L.rnnoise_batch_debug_set_frame_counter.argtypes = [vp, C.c_longlong]
        L.rnnoise_batch_get_streams.restype = ip; L.rnnoise_batch_get_streams.argtypes = [vp]
        L.rnnoise_batch_get_lanes.restype = ip; L.rnnoise_batch_get_lanes.argtypes = [vp]
        L.rnnoise_process_frame_batch.restype = ip; L.rnnoise_process_frame_batch.argtypes = [vp, vp, vp, vp]
        L.rnnoise_process_frame_batch_async.restype = ip; L.rnnoise_process_frame_batch_async.argtypes = [vp, vp, vp, vp]
        for nm in ("rnnoise_process_frame_batch_s16", "rnnoise_process_frame_batch_s16_async", "rnnoise_process_frame_batch_device_s16"):
            getattr(L, nm).restype = ip; getattr(L, nm).argtypes = [vp, vp, vp, vp]
        for nm in ("rnnoise_process_frames_batch", "rnnoise_process_frames_batch_s16", "rnnoise_process_frames_batch_device",
                   "rnnoise_process_frames_batch_device_s16"):
            getattr(L, nm).restype = ip; getattr(L, nm).argtypes = [vp, vp, vp, vp, ip]
        for nm in ("rnnoise_batch_train_features", "rnnoise_batch_train_features_device"):
            getattr(L, nm).restype = ip; getattr(L, nm).argtypes = [vp] * 8
        L.rnnoise_process_frame_batch_device.restype = ip; L.rnnoise_process_frame_batch_device.argtypes = [vp, vp, vp, vp]
        L.rnnoise_batch_prefilter_device.restype = ip; L.rnnoise_batch_prefilter_device.argtypes = [vp, vp]
        L.rnnoise_batch_sync.restype = ip; L.rnnoise_batch_sync.argtypes = [vp]
        L.rnnoise_batch_set_stream.restype = ip; L.rnnoise_batch_set_stream.argtypes = [vp, vp]
        L.rnnoise_batch_reset_stream.restype = ip; L.rnnoise_batch_reset_stream.argtypes = [vp, ip]
        L.rnnoise_batch_launches_per_frame.restype = ip; L.rnnoise_batch_launches_per_frame.argtypes = [vp]
        L.rnnoise_batch_profile.restype = ip; L.rnnoise_batch_profile.argtypes = [vp, ip]
        L.rnnoise_batch_profile_read.restype = ip
        L.rnnoise_batch_profile_read.argtypes = [vp, fp, C.POINTER(C.c_char_p), ip, C.POINTER(ip)]
        L.rnnoise_batch_timeline_read.restype = ip; L.rnnoise_batch_timeline_read.argtypes = [vp, fp, ip]
        L.rnnoise_batch_debug_read.restype = ip; L.rnnoise_batch_debug_read.argtypes = [vp, ip, ip, fp, ip]
        L.rnnoise_batch_debug_read_all.restype = ip; L.rnnoise_batch_debug_read_all.argtypes = [vp, ip, fp, ip]
        _lib = L
    return _lib


class Model:
    """RNNModel* (rnnoise_model_from_filename / rnnoise_model_from_buffer)."""

    def __init__(self, path=None, buffer=None):
        L = lib()
        self._buf = None
        if path is not None:
            self.handle = L.rnnoise_model_from_filename(os.fsencode(path))
        else:
            self._buf = bytes(buffer)  # must outlive the model (borrowed, like the reference)
            self.handle = L.rnnoise_model_from_buffer(self._buf, len(self._buf))
        if not self.handle:
            raise ValueError("not a valid RNNoise weight blob")

    def free(self):
        if self.handle:
            lib().rnnoise_model_free(self.handle)
            self.handle = None


class Batch:
    """RNNoiseBatch*: nb_streams independent denoiser states resident on one GPU, or -- with `devices`, a list
    of CUDA device indices -- sharded over several GPUs of one box (rnnoise_batch_create_multi)."""

    def __init__(self, model, nb_streams, device=0, devices=None):
        self.model = model
        self.nb_streams = nb_streams
        if devices is None:
            self.handle = lib().rnnoise_batch_create(model.handle, nb_streams, device)
        else:
            arr = (C.c_int * len(devices))(*devices)
            self.handle = lib().rnnoise_batch_create_multi(model.handle, nb_streams, arr, len(devices))
        if not self.handle:
            raise RuntimeError("rnnoise_batch_create failed (no usable CUDA device, bad model or out of memory)")
        self.lanes = lib().rnnoise_batch_get_lanes(self.handle)
        self.nb_devices = lib().rnnoise_batch_get_devices(self.handle)

    def shard(self, k):
        """-> (cuda device, first stream, stream count) of shard k."""
        d, f, n = C.c_int(), C.c_int(), C.c_int()
        if lib().rnnoise_batch_get_shard(self.handle, k, C.byref(d), C.byref(f), C.byref(n)) != 0:
            raise IndexError(k)
        return d.value, f.value, n.value

    @staticmethod
    def _ptrs(lst):
        return None if lst is None else (C.c_void_p * len(lst))(*lst)

    def process_device_multi(self, d_out, d_in, d_vad=None):
        """Lists of device pointers (ints), one per device of the batch; asynchronous."""
        if lib().rnnoise_process_frame_batch_device_multi(self.handle, self._ptrs(d_out), self._ptrs(d_in), self._ptrs(d_vad)) != 0:
            raise RuntimeError("rnnoise_process_frame_batch_device_multi failed")

    def prefilter_device_multi(self, d_in_next):
        if lib().rnnoise_batch_prefilter_device_multi(self.handle, self._ptrs(d_in_next)) != 0:
            raise RuntimeError("rnnoise_batch_prefilter_device_multi failed")

    def set_stream_multi(self, streams):
        if lib().rnnoise_batch_set_stream_multi(self.handle, self._ptrs(streams)) != 0:
            raise RuntimeError("rnnoise_batch_set_stream_multi failed")

    def debug_set_frame_counter(self, frames):
        if lib().rnnoise_batch_debug_set_frame_counter(self.handle, int(frames)) != 0:
            raise RuntimeError("rnnoise_batch_debug_set_frame_counter failed (batch not fresh)")

    def process(self, pcm, want_vad=True):
        """pcm: float32 [nb_streams][480] host array -> (out [nb_streams][480], vad [nb_streams])."""
        x = np.ascontiguousarray(pcm, np.float32)
        assert x.shape == (self.nb_streams, FRAME_SIZE)
        out = np.empty_like(x)
        vad = np.empty(self.nb_streams, np.float32)
        rc = lib().rnnoise_process_frame_batch(self.handle, out.ctypes.data, x.ctypes.data, vad.ctypes.data)
        if rc != 0:
            raise RuntimeError("rnnoise_process_frame_batch failed")
        return out, vad

    def process_ptr(self, out_ptr, in_ptr, vad_ptr=None):
        """Host-buffer call on raw addresses (e.g. pinned torch tensors)."""
        if lib().rnnoise_process_frame_batch(self.handle, out_ptr, in_ptr, vad_ptr) != 0:
            raise RuntimeError("rnnoise_process_frame_batch failed")

    def process_s16(self, pcm16):
        """pcm16: int16 [nb_streams][480] host array -> (out int16 [nb_streams][480], vad)."""
        x = np.ascontiguousarray(pcm16, np.int16)
        assert x.shape == (self.nb_streams, FRAME_SIZE)
        out = np.empty_like(x)
        vad = np.empty(self.nb_streams, np.float32)
        if lib().rnnoise_process_frame_batch_s16(self.handle, out.ctypes.data, x.ctypes.data, vad.ctypes.data) != 0:
            raise RuntimeError("rnnoise_process_frame_batch_s16 failed")
        return out, vad

    def process_frames(self, pcm):
        """Multi-frame call: pcm [nb_streams][T * 480] float32 or int16 host array (each stream's audio
        contiguous) -> (out, same shape and dtype; vad float32 [nb_streams][T])."""
        s16 = np.asarray(pcm).dtype == np.int16
        x = np.ascontiguousarray(pcm, np.int16 if s16 else np.float32)
        assert x.ndim == 2 and x.shape[0] == self.nb_streams and x.shape[1] % FRAME_SIZE == 0 and x.shape[1] > 0
        T = x.shape[1] // FRAME_SIZE
        out = np.empty_like(x)
        vad = np.empty((self.nb_streams, T), np.float32)
        fn = lib().rnnoise_process_frames_batch_s16 if s16 else lib().rnnoise_process_frames_batch
        if fn(self.handle, out.ctypes.data, x.ctypes.data, vad.ctypes.data, T) != 0:
            raise RuntimeError("rnnoise_process_frames_batch failed")
        return out, vad

    def process_frames_device(self, d_out, d_in, d_vad, nb_frames, s16=False):
        """Device pointers (ints) to [nb_streams][nb_frames * 480] buffers; asynchronous."""
        fn = lib().rnnoise_process_frames_batch_device_s16 if s16 else lib().rnnoise_process_frames_batch_device
        if fn(self.handle, d_out, d_in, d_vad, nb_frames) != 0:
            raise RuntimeError("rnnoise_process_frames_batch_device failed")

    def train_features(self, clean, noisy, vad_target=None, noise_free=None, lowpass=None, band_lp=None):
        """Training-feature records (include/rnnoise.h: rnnoise_batch_train_features): clean, noisy float32
        [nb_streams][480]; optional per-stream arrays -> float32 [nb_streams][98] = features | g | vad target."""
        c = np.ascontiguousarray(clean, np.float32); n = np.ascontiguousarray(noisy, np.float32)
        assert c.shape == n.shape == (self.nb_streams, FRAME_SIZE)
        keep = [None if a is None else np.ascontiguousarray(a, dt) for a, dt in
                ((vad_target, np.float32), (noise_free, np.int32), (lowpass, np.int32), (band_lp, np.int32))]
        assert all(a is None or a.shape == (self.nb_streams,) for a in keep)
        rec = np.empty((self.nb_streams, 98), np.float32)
        if lib().rnnoise_batch_train_features(self.handle, rec.ctypes.data, c.ctypes.data, n.ctypes.data,
                                              *[None if a is None else a.ctypes.data for a in keep]) != 0:
            raise RuntimeError("rnnoise_batch_train_features failed")
        return rec

    def process_ptr_s16_async(self, out_ptr, in_ptr, vad_ptr=None):
        if lib().rnnoise_process_frame_batch_s16_async(self.handle, out_ptr, in_ptr, vad_ptr) != 0:
            raise RuntimeError("rnnoise_process_frame_batch_s16_async failed")

    def process_ptr_async(self, out_ptr, in_ptr, vad_ptr=None):
        """Pipelined host-buffer call (pinned memory); results valid after sync()."""
        if lib().rnnoise_process_frame_batch_async(self.handle, out_ptr, in_ptr, vad_ptr) != 0:
            raise RuntimeError("rnnoise_process_frame_batch_async failed")

    def process_device(self, d_out, d_in, d_vad=None):
        """Device pointers (ints); asynchronous on the batch's stream."""
        if lib().rnnoise_process_frame_batch_device(self.handle, d_out, d_in, d_vad) != 0:
            raise RuntimeError("rnnoise_process_frame_batch_device failed")

    def prefilter_device(self, d_in_next):
        """Pipelining hint: start the next frame's high-pass prefilter now (see include/rnnoise.h)."""
        if lib().rnnoise_batch_prefilter_device(self.handle, d_in_next) != 0:
            raise RuntimeError("rnnoise_batch_prefilter_device failed")

    def timeline(self, max_frames=256):
        """[frames][8] stage-boundary times in ms ($RNNOISE_B200_TIMELINE must be set when the batch is created)."""
        buf = np.zeros((max_frames, 8), np.float32)
        n = lib().rnnoise_batch_timeline_read(self.handle, buf.ctypes.data_as(C.POINTER(C.c_float)), buf.size)
        if n < 0:
            raise RuntimeError("rnnoise_batch_timeline_read failed")
        return buf[:n]

    def set_stream(self, cuda_stream):
        if lib().rnnoise_batch_set_stream(self.handle, cuda_stream) != 0:
            raise RuntimeError("rnnoise_batch_set_stream failed")

    def sync(self):
        if lib().rnnoise_batch_sync(self.handle) != 0:
            raise RuntimeError("rnnoise_batch_sync failed")

    def reset_stream(self, s):
        if lib().rnnoise_batch_reset_stream(self.handle, s) != 0:
            raise RuntimeError("rnnoise_batch_reset_stream failed")

    @property
    def launches_per_frame(self):
        return lib().rnnoise_batch_launches_per_frame(self.handle)

    def profile(self, enable):
        if lib().rnnoise_batch_profile(self.handle, 1 if enable else 0) != 0:
            raise RuntimeError("rnnoise_batch_profile failed")

    def profile_read(self):
        """-> (dict kernel name -> total ms, frames profiled)"""
        cap = 32
        ms = (C.c_float * cap)(); names = (C.c_char_p * cap)(); frames = C.c_int(0)
        n = lib().rnnoise_batch_profile_read(self.handle, ms, names, cap, C.byref(frames))
        if n <= 0:
            raise RuntimeError("rnnoise_batch_profile_read failed")
        return {names[i].decode(): float(ms[i]) for i in range(n)}, frames.value

    def debug(self, what, stream):
        buf = np.empty(2048, np.float32)
        n = lib().rnnoise_batch_debug_read(self.handle, DBG[what], stream, buf.ctypes.data_as(C.POINTER(C.c_float)), buf.size)
        if n < 0:
            raise RuntimeError("debug_read failed")
        return buf[:n].copy()

    def debug_all(self, what):
        """Item `what` (pitch, silence, features, gains) of every stream -> float32 [nb_streams][n]."""
        n = dict(pitch=2, silence=1, features=65, gains=32)[what]
        buf = np.empty((self.nb_streams, n), np.float32)
        if lib().rnnoise_batch_debug_read_all(self.handle, DBG[what], buf.ctypes.data_as(C.POINTER(C.c_float)), buf.size) != n:
            raise RuntimeError("debug_read_all failed")
        return buf

    def destroy(self):
        if self.handle:
            lib().rnnoise_batch_destroy(self.handle)
            self.handle = None
