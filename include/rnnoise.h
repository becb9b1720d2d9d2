/* rnnoise.h -- public C ABI of the H100-native batched denoise engine (librnnoise_b200.so).
 *
 * Drop-in surface of xiph/rnnoise's include/rnnoise.h (reference file:line cited per entry point)
 * plus the batched entry points the GPU engine adds.  Plain C linkage, plain pointers and sizes,
 * no CUDA or torch types in any signature.  Every entry point that computes runs on the GPU; there
 * is no CPU fallback: creation fails (NULL / -1) when no CUDA device is usable.
 *
 * Data conventions (unchanged from the reference, examples/rnnoise_demo.c:52-61): mono 48 kHz,
 * 480 samples per frame, float samples in int16 units (+-32768, not +-1); `out` may alias `in`.
 */
#ifndef RNNOISE_H
#define RNNOISE_H 1

#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef RNNOISE_EXPORT
# if defined(__GNUC__) && defined(RNNOISE_BUILD)
#  define RNNOISE_EXPORT __attribute__ ((visibility ("default")))
# else
#  define RNNOISE_EXPORT
# endif
#endif

typedef struct DenoiseState DenoiseState;
typedef struct RNNModel RNNModel;
typedef struct RNNoiseBatch RNNoiseBatch;

/* ------------------------------------------------------------------------------------------ */
/* Reference surface (single stream).  Each DenoiseState is one stream of a private batch of 1, */
/* driven through exactly the same kernels as the batched path.                                  */
/* ------------------------------------------------------------------------------------------ */

/** Size of DenoiseState in bytes.  Replaces reference include/rnnoise.h:57 (src/denoise.c:277). */
RNNOISE_EXPORT int rnnoise_get_size(void);

/** Samples per rnnoise_process_frame() call (480).  Replaces rnnoise.h:62 (denoise.c:281). */
RNNOISE_EXPORT int rnnoise_get_frame_size(void);

/** Initialise caller-provided memory of rnnoise_get_size() bytes.  Returns 0, or -1 when the model
 *  blob lacks/mis-sizes an array (same rule as src/parse_lpcnet_weights.c:123-176) or no GPU is
 *  usable.  Replaces rnnoise.h:71 (denoise.c:285).  Device resources attached to a state
 *  initialised this way are released by rnnoise_destroy_inplace() (or at process exit).
 *  model == NULL selects the built-in model; this build has no built-in weights (the reference
 *  downloads them, download_model.sh:4-31), so the blob named by $RNNOISE_B200_DEFAULT_MODEL is
 *  loaded instead and -1 is returned when that is unset or unreadable. */
RNNOISE_EXPORT int rnnoise_init(DenoiseState *st, RNNModel *model);

/** Allocate + initialise.  NULL on failure.  Replaces rnnoise.h:80 (denoise.c:311). */
RNNOISE_EXPORT DenoiseState *rnnoise_create(RNNModel *model);

/** Free a state made by rnnoise_create().  Replaces rnnoise.h:87 (denoise.c:323). */
RNNOISE_EXPORT void rnnoise_destroy(DenoiseState *st);

/** Release the device side of a state set up with rnnoise_init() on caller memory (new). */
RNNOISE_EXPORT void rnnoise_destroy_inplace(DenoiseState *st);

/** Denoise one 480-sample frame; returns the VAD probability (0 on a silent frame).
 *  Replaces rnnoise.h:94 (denoise.c:457). */
RNNOISE_EXPORT float rnnoise_process_frame(DenoiseState *st, float *out, const float *in);

/** Model from a memory buffer (borrowed; must outlive the model).  NULL when the buffer is not a
 *  well-formed weight blob.  Replaces rnnoise.h:102 (denoise.c:235). */
RNNOISE_EXPORT RNNModel *rnnoise_model_from_buffer(const void *ptr, int len);

/** Model from an open FILE (contents are copied; the FILE stays the caller's).
 *  Replaces rnnoise.h:111 (denoise.c:252). */
RNNOISE_EXPORT RNNModel *rnnoise_model_from_file(FILE *f);

/** Model from a file name; NULL when it cannot be opened (the reference dereferences the failed
 *  fopen, denoise.c:246-248).  Replaces rnnoise.h:118 (denoise.c:244). */
RNNOISE_EXPORT RNNModel *rnnoise_model_from_filename(const char *filename);

/** Free a model (after every state/batch using it).  Replaces rnnoise.h:125 (denoise.c:271). */
RNNOISE_EXPORT void rnnoise_model_free(RNNModel *model);

/* ------------------------------------------------------------------------------------------ */
/* Batched surface (new; named by the north star).  One RNNoiseBatch = nb_streams independent     */
/* DenoiseStates resident in the HBM of ONE device, advanced in lock-step: one call = one 10 ms   */
/* frame of every stream.  Streams never interact; multi-GPU use is one batch per device.        */
/* ------------------------------------------------------------------------------------------ */

/** Create nb_streams zero-initialised stream states on CUDA device `device` (>= 0).
 *  NULL on failure (bad model, nb_streams < 1, no such device, out of memory). */
RNNOISE_EXPORT RNNoiseBatch *rnnoise_batch_create(RNNModel *model, int nb_streams, int device);

/** Multi-device batch (SURVEY section 8e): nb_streams stream states sharded over the nb_devices CUDA devices
 *  listed in devices[] as contiguous stream ranges (shard k = streams [k*S/G, (k+1)*S/G), remainders to the
 *  first shards), one host thread driving all of them.  Streams never interact, so there is no collective:
 *  every per-frame call fans out over the devices asynchronously and rnnoise_batch_sync() joins them.  The
 *  host-buffer entry points (rnnoise_process_frame_batch{,_async,_s16,...}, rnnoise_process_frames_batch*,
 *  rnnoise_batch_train_features) work unchanged on [nb_streams][...] host buffers; device-resident audio goes
 *  through the *_multi forms below, one pointer per device.  NULL on failure. */
RNNOISE_EXPORT RNNoiseBatch *rnnoise_batch_create_multi(RNNModel *model, int nb_streams, const int *devices, int nb_devices);
/** Number of devices of a batch, and shard k: its CUDA device, first stream and stream count.  0 / -1. */
RNNOISE_EXPORT int rnnoise_batch_get_devices(const RNNoiseBatch *b);
RNNOISE_EXPORT int rnnoise_batch_get_shard(const RNNoiseBatch *b, int k, int *device, int *first_stream, int *nb_streams);
/** Device-pointer frame call of a multi-device batch: d_in[k] / d_out[k] ([shard streams][480]) and d_vad[k]
 *  ([shard streams]; the array or single entries may be NULL) live on device k.  Enqueues and returns.
 *  rnnoise_batch_prefilter_device_multi / rnnoise_batch_set_stream_multi are the per-device forms of the
 *  calls below (streams[k] = a cudaStream_t of device k).  All also accept a single-device batch. */
RNNOISE_EXPORT int rnnoise_process_frame_batch_device_multi(RNNoiseBatch *b, float *const *d_out, const float *const *d_in, float *const *d_vad);
RNNOISE_EXPORT int rnnoise_batch_prefilter_device_multi(RNNoiseBatch *b, const float *const *d_in_next);
RNNOISE_EXPORT int rnnoise_batch_set_stream_multi(RNNoiseBatch *b, void *const *streams);

RNNOISE_EXPORT void rnnoise_batch_destroy(RNNoiseBatch *b);

/* Error discipline of every per-frame call below: arguments and call-order preconditions are checked on the
 * whole batch before anything is enqueued -- such a -1 leaves the batch untouched.  A -1 caused by a CUDA error
 * while the frame was being enqueued cannot be undone (parts of the batch are a frame ahead): the batch is
 * poisoned, every later per-frame call returns -1, and the only valid operation is rnnoise_batch_destroy(). */

RNNOISE_EXPORT int rnnoise_batch_get_streams(const RNNoiseBatch *b);
/** Inside a device batch the DSP stages of a frame (analysis front, output tail) run as 1..4 "lanes" -- sub-grids over
 *  contiguous stream ranges on their own CUDA streams -- while the network runs once over the whole batch; streams are
 *  independent, so results do not depend on the split.  The default (two lanes from 1024 up to 32767 streams, else one)
 *  can be overridden with $RNNOISE_B200_LANES at creation time.  Returns the number of lanes. */
RNNOISE_EXPORT int rnnoise_batch_get_lanes(const RNNoiseBatch *b);

/** Host-buffer call: in/out are [nb_streams][480] floats in host memory (pinned memory makes the
 *  copies asynchronous DMA), vad is [nb_streams] (may be NULL).  Copies in, runs the frame, copies
 *  out, and returns after the results are in `out`/`vad`.  0 on success, -1 on a CUDA error. */
RNNOISE_EXPORT int rnnoise_process_frame_batch(RNNoiseBatch *b, float *out, const float *in, float *vad);

/** Pipelined host-buffer call: same arguments as rnnoise_process_frame_batch() but returns as soon
 *  as the frame is enqueued.  The H2D copy, the kernels and the D2H copy of consecutive calls run on
 *  three streams over double-buffered staging, so copy-in(n+1), compute(n) and copy-out(n-1) overlap.
 *  `in` must stay valid and `out`/`vad` must not be read until rnnoise_batch_sync() (or a later
 *  synchronous call) returns.  Use pinned host memory, otherwise the copies serialise. */
RNNOISE_EXPORT int rnnoise_process_frame_batch_async(RNNoiseBatch *b, float *out, const float *in, float *vad);

/** 16-bit PCM variants (SURVEY section 8f rank 1): in/out are [nb_streams][480] int16 samples, the
 *  format examples/rnnoise_demo.c:53-58 reads and writes.  Input samples are widened to float exactly
 *  (x = tmp[i]); output samples are narrowed like the demo's C cast (truncation toward zero, low 16
 *  bits).  Half the PCIe bytes of the float calls; same kernels otherwise.  The _async form pipelines
 *  like rnnoise_process_frame_batch_async(); the _device form takes device pointers. */
RNNOISE_EXPORT int rnnoise_process_frame_batch_s16(RNNoiseBatch *b, short *out, const short *in, float *vad);
RNNOISE_EXPORT int rnnoise_process_frame_batch_s16_async(RNNoiseBatch *b, short *out, const short *in, float *vad);
RNNOISE_EXPORT int rnnoise_process_frame_batch_device_s16(RNNoiseBatch *b, short *d_out, const short *d_in, float *d_vad);

/** Multi-frame calls (SURVEY section 8f rank 2): nb_frames consecutive 10 ms frames of every stream in
 *  one call -- offline / file denoising, where the reference loops rnnoise_process_frame over a file
 *  (examples/rnnoise_demo.c:53-64).  Each stream's audio is contiguous: in/out are
 *  [nb_streams][nb_frames * 480] samples, vad is [nb_streams][nb_frames] (may be NULL).  out may alias
 *  in.  The result is bit-identical to nb_frames frame-at-a-time calls.  Host forms block until out/vad
 *  are complete; they move the audio in chunks ($RNNOISE_B200_MULTI_CHUNK frames, default 16) through
 *  double-buffered device staging so copies overlap the kernels (pinned host memory recommended).
 *  The _device form takes device pointers, enqueues on the batch's stream and returns. */
RNNOISE_EXPORT int rnnoise_process_frames_batch(RNNoiseBatch *b, float *out, const float *in, float *vad, int nb_frames);
RNNOISE_EXPORT int rnnoise_process_frames_batch_s16(RNNoiseBatch *b, short *out, const short *in, float *vad, int nb_frames);
RNNOISE_EXPORT int rnnoise_process_frames_batch_device(RNNoiseBatch *b, float *d_out, const float *d_in, float *d_vad, int nb_frames);
RNNOISE_EXPORT int rnnoise_process_frames_batch_device_s16(RNNoiseBatch *b, short *d_out, const short *d_in, float *d_vad, int nb_frames);

/** Training-feature extraction (SURVEY section 8f rank 4): the per-frame body of the reference's
 *  training-data tool, src/dump_features.c:466-491 (a -DTRAINING=1 build), for every stream of the batch:
 *    rnn_frame_analysis(clean state, Y, Ey, clean)                     (denoise.c:332-345)
 *    quiet = rnn_compute_frame_features(noisy state, X, P, Ex, Ep, Exp, features, noisy)   (:347-398)
 *    g[i] = min(1, sqrt((Ey[i] + 1e-3) / (Ex[i] + 1e-3))), or -1 where the target is undefined
 *  with the TRAINING semantics: X and Y low-passed at lowpass[s] bins (:340-343), no silence
 *  short-circuit (:389), quiet = E < 0.1 (:397).  clean/noisy are [nb_streams][480] floats, already
 *  mixed and filtered by the caller (the tool's sequence-level filtering and mixing, :411-463, stay on the
 *  host); rec is [nb_streams][RNNOISE_TRAIN_RECORD] = features[65] | g[32] | vad_target, the record
 *  dump_features writes (:487-489).  vad_target [nb_streams] floats, noise_free [nb_streams] ints (non-zero:
 *  noise_gain == 0 && fgnoise_gain == 0, :477), lowpass / band_lp [nb_streams] ints (:400-406); any of the
 *  four may be NULL (0, 0, 481, 32).  The batch keeps the two signal histories (clean and noisy) per
 *  stream; use a batch either for this or for denoising, not both.  0 on success, -1 on error. */
#define RNNOISE_TRAIN_RECORD 98
RNNOISE_EXPORT int rnnoise_batch_train_features(RNNoiseBatch *b, float *rec, const float *clean, const float *noisy,
                                                const float *vad_target, const int *noise_free, const int *lowpass, const int *band_lp);
RNNOISE_EXPORT int rnnoise_batch_train_features_device(RNNoiseBatch *b, float *d_rec, const float *d_clean, const float *d_noisy,
                                                       const float *d_vad_target, const int *d_noise_free, const int *d_lowpass,
                                                       const int *d_band_lp);

/** Device-buffer call: d_in/d_out/d_vad are device pointers on the batch's device (d_out may alias
 *  d_in; d_vad may be NULL).  Enqueues the frame on the batch's stream and returns without
 *  synchronising.  0 on success, -1 on a launch error. */
RNNOISE_EXPORT int rnnoise_process_frame_batch_device(RNNoiseBatch *b, float *d_out, const float *d_in, float *d_vad);

/** Optional pipelining hint for the device-buffer path: d_in_next (already complete in device memory)
 *  is the input of the next frame that has not been handed to rnnoise_process_frame_batch_device()
 *  yet.  Its high-pass prefilter (the only stage that depends on nothing but the input and the previous
 *  prefilter) is started right away on an internal stream, overlapping the frame in flight; the
 *  following rnnoise_process_frame_batch_device() call must pass the same pointer.  At most two frames
 *  ahead.  0 / -1. */
RNNOISE_EXPORT int rnnoise_batch_prefilter_device(RNNoiseBatch *b, const float *d_in_next);

/** Block until everything enqueued on the batch's stream has finished.  0 / -1. */
RNNOISE_EXPORT int rnnoise_batch_sync(RNNoiseBatch *b);

/** Order the batch's device-pointer calls with an existing CUDA stream (a cudaStream_t passed as void*), so callers
 *  can pipeline their own work and time with events on that stream.  The batch keeps its private streams (analysis
 *  front, network, output tail run side by side across consecutive frames): the kernels of a call that read the input
 *  or write out/vad start after the work already enqueued on the caller's stream, and the caller's stream waits for the
 *  call's completion, so the call behaves like work on that one stream.  NULL detaches. */
RNNOISE_EXPORT int rnnoise_batch_set_stream(RNNoiseBatch *b, void *cuda_stream);

/** Re-zero the state of one stream (what rnnoise_init() does to a DenoiseState): ordered after every frame
 *  already handed to the batch, synchronises.  Fails (-1) while a rnnoise_batch_prefilter_device() hint is
 *  pending, because that hint has already filtered the next frame with the old state.  0 / -1. */
RNNOISE_EXPORT int rnnoise_batch_reset_stream(RNNoiseBatch *b, int stream);

/** Number of kernel launches one rnnoise_process_frame_batch_device() call issues. */
RNNOISE_EXPORT int rnnoise_batch_launches_per_frame(const RNNoiseBatch *b);

/** Per-kernel timing for roofline reports.  enable != 0: every following frame records CUDA events
 *  around each kernel launch on the batch's stream and accumulates the elapsed times (the call then
 *  synchronises after each frame).  enable == 0 stops.  Accumulators reset on every enable. */
RNNOISE_EXPORT int rnnoise_batch_profile(RNNoiseBatch *b, int enable);

/** Reads the accumulators: ms[i] = total milliseconds spent in kernel i over *frames frames,
 *  i < rnnoise_batch_launches_per_frame().  names[i] (optional) receives static strings.
 *  Returns the number of kernels or -1. */
RNNOISE_EXPORT int rnnoise_batch_profile_read(RNNoiseBatch *b, float *ms, const char **names, int capacity, int *frames);

/* ------------------------------------------------------------------------------------------ */
/* Introspection for parity tests (device -> host copies of per-stream intermediates of the last */
/* processed frame).  Not needed by applications.                                                */
/* ------------------------------------------------------------------------------------------ */
enum {
  RNNOISE_DBG_FEATURES = 0,   /* [65]  features fed to the network (denoise.c:347 output)        */
  RNNOISE_DBG_X = 1,          /* [962] analysis spectrum X, interleaved re/im                    */
  RNNOISE_DBG_P = 2,          /* [962] pitch spectrum P                                          */
  RNNOISE_DBG_EX = 3,         /* [32]  band energies of X                                        */
  RNNOISE_DBG_EP = 4,         /* [32]                                                            */
  RNNOISE_DBG_EXP = 5,        /* [32]  normalised band correlation                               */
  RNNOISE_DBG_GAINS = 6,      /* [32]  raw network gains g (before denoise.c:483)               */
  RNNOISE_DBG_LASTG = 7,      /* [32]  st->lastg                                                 */
  RNNOISE_DBG_XB = 8,         /* [480] input after the high-pass biquad                          */
  RNNOISE_DBG_GRU1 = 9,       /* [gru] GRU states after the frame                               */
  RNNOISE_DBG_GRU2 = 10,
  RNNOISE_DBG_GRU3 = 11,
  RNNOISE_DBG_CONV1_STATE = 12, /* [130] */
  RNNOISE_DBG_CONV2_STATE = 13, /* [2*cond] conv2 memory as the u8 values 127 + rne(127 x) it is kept in */
  RNNOISE_DBG_PITCH = 14,     /* [2]   {last_period (as float), last_gain}                       */
  RNNOISE_DBG_SILENCE = 15,   /* [1]   1.0 when the frame was classified silent                  */
  RNNOISE_DBG_CONV2_OUT = 16  /* [gru] conv2 output of the frame                                */
};
/** Pipeline timeline (diagnostics): with $RNNOISE_B200_TIMELINE=N set at batch creation, the first N frames
 *  record timing events at the stage boundaries.  Synchronises, then writes [frames][8] milliseconds since
 *  the first point: H2D start, H2D end, prefilter end, pitch end, spectrum end, network start, synthesis end,
 *  D2H end (NaN where a stage did not run through this call path).  Returns the frames written, -1 on error. */
RNNOISE_EXPORT int rnnoise_batch_timeline_read(RNNoiseBatch *b, float *ms, int capacity);

/** Test hook: start a fresh batch (nothing processed yet) at frame index `frames`, so that tests can cross the
 *  wrap of the internal frame counter within a few frames.  0 / -1. */
RNNOISE_EXPORT int rnnoise_batch_debug_set_frame_counter(RNNoiseBatch *b, long long frames);

/** Copies item `what` of stream `stream` into dst (capacity in floats); returns the number of
 *  floats written or -1. */
RNNOISE_EXPORT int rnnoise_batch_debug_read(RNNoiseBatch *b, int what, int stream, float *dst, int capacity);

/** Bulk form for long parity statistics: item `what` (RNNOISE_DBG_PITCH, _SILENCE, _FEATURES or _GAINS) of every
 *  stream into dst as [nb_streams][n] floats; capacity must be exactly nb_streams * n (n = 2, 1, 65, 32).
 *  Returns n or -1. */
RNNOISE_EXPORT int rnnoise_batch_debug_read_all(RNNoiseBatch *b, int what, float *dst, int capacity);

#ifdef __cplusplus
}
#endif

#endif
