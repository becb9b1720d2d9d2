/* rnnoise_api.c -- the public C ABI of include/rnnoise.h, in plain C, on top of the CUDA engine.
 *
 * Mirrors the reference's API implementation (src/denoise.c:227-325, 457-504) entry point by entry
 * point; the arithmetic itself lives in the CUDA kernels (engine.cu).  There is no CPU path: every
 * creation call fails when the engine cannot be brought up on a GPU.
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/rnnoise.h"
#include "engine.h"
#include "model_blob.h"

#define FRAME_SIZE 480
#define STATE_MAGIC 0x42323030 /* "B200" */

struct RNNModel {
  const void *const_blob; /* borrowed (from_buffer) */
  void *blob;             /* owned (from_file / from_filename) */
  int blob_len;
  B200HostModel host;     /* parsed + dense-expanded; valid iff parsed != 0 */
  int parsed;
};

/* A batch is one engine per device (rnnoise_batch_create_multi shards the streams contiguously over the devices; the
 * plain rnnoise_batch_create is the one-device case).  Inside an engine the DSP stages of a frame run as 1..4 sub-grids
 * ("lanes": contiguous stream ranges on their own CUDA streams) while the network runs once over the whole device batch
 * (engine.cu); streams never interact, so results do not depend on any of these splits.  $RNNOISE_B200_LANES overrides
 * the lane count.  `lanes` below counts ENGINES (= devices). */
#define B200_MAX_DEVICES 16
#define B200_MAX_ENGINES B200_MAX_DEVICES
struct RNNoiseBatch {
  int lanes;                       /* engines = devices */
  int first[B200_MAX_ENGINES + 1]; /* engine l owns streams [first[l], first[l + 1]) */
  B200Engine *engine[B200_MAX_ENGINES];
  int nb_streams;
  int nb_devices;
  int device[B200_MAX_DEVICES];
  int dev_lane[B200_MAX_DEVICES + 1];   /* = k: kept so that shard bookkeeping reads the same for 1 or more engines per device */
  /* set when a per-frame call failed after some engines had already enqueued the frame: they are then out of step with
   * each other for good, so every later call fails cleanly instead of producing skewed audio */
  int poisoned;
  /* multi-device batches: one host worker thread per device, so that the enqueue cost of a frame (copies, launches,
   * event operations on the host-buffer path) is paid in parallel instead of G times in a row by the caller's thread,
   * where it would exceed the GPU step with several devices.  A call posts one job per device and returns when all of them are ENQUEUED. */
  struct Worker *workers;
};

typedef struct Job {
  int kind;                 /* J_* */
  void *out; const void *in; float *vad;
  int T, s16;
} Job;
enum { J_HOST_ASYNC = 1, J_DEVICE, J_PREFILTER, J_SYNC, J_FRAMES_HOST };
typedef struct Worker {
  pthread_t th;
  pthread_mutex_t mu;
  pthread_cond_t cv;
  int state;                /* 0 idle, 1 job posted, 2 done, -1 quit */
  Job job;
  int rc;
  B200Engine *e;
} Worker;

static int run_job(B200Engine *e, const Job *j) {
  switch (j->kind) {
    case J_HOST_ASYNC:
      return j->s16 ? b200_engine_frame_host_async_s16(e, (short *)j->out, (const short *)j->in, j->vad)
                    : b200_engine_frame_host_async(e, (float *)j->out, (const float *)j->in, j->vad);
    case J_DEVICE:
      return j->s16 ? b200_engine_frame_device_s16(e, (short *)j->out, (const short *)j->in, j->vad)
                    : b200_engine_frame_device(e, (float *)j->out, (const float *)j->in, j->vad);
    case J_PREFILTER: return b200_engine_prefilter_device(e, (const float *)j->in);
    case J_SYNC: return b200_engine_sync(e);
    case J_FRAMES_HOST: return b200_engine_frames_host_enqueue(e, j->out, j->in, j->vad, j->T, j->s16, j->T);
  }
  return -1;
}
static void *worker_main(void *arg) {
  Worker *w = (Worker *)arg;
  pthread_mutex_lock(&w->mu);
  for (;;) {
    while (w->state != 1 && w->state != -1) pthread_cond_wait(&w->cv, &w->mu);
    if (w->state == -1) break;
    pthread_mutex_unlock(&w->mu);
    w->rc = run_job(w->e, &w->job);
    pthread_mutex_lock(&w->mu);
    w->state = 2;
    pthread_cond_broadcast(&w->cv);
  }
  pthread_mutex_unlock(&w->mu);
  return NULL;
}
/* runs jobs[l] on engine l for every engine: on the worker threads when the batch has them, else in place.
 * Returns 0, or -1 if any job failed (all jobs are always run to completion). */
static int run_jobs(RNNoiseBatch *b, const Job *jobs) {
  int l, rc = 0;
  if (!b->workers) {
    for (l = 0; l < b->lanes; l++) rc |= run_job(b->engine[l], &jobs[l]);
    return rc ? -1 : 0;
  }
  for (l = 0; l < b->lanes; l++) {
    Worker *w = &b->workers[l];
    pthread_mutex_lock(&w->mu);
    w->job = jobs[l];
    w->state = 1;
    pthread_cond_broadcast(&w->cv);
    pthread_mutex_unlock(&w->mu);
  }
  for (l = 0; l < b->lanes; l++) {
    Worker *w = &b->workers[l];
    pthread_mutex_lock(&w->mu);
    while (w->state != 2) pthread_cond_wait(&w->cv, &w->mu);
    w->state = 0;
    rc |= w->rc;
    pthread_mutex_unlock(&w->mu);
  }
  return rc ? -1 : 0;
}
#define LANE_COUNT(b, l) ((b)->first[(l) + 1] - (b)->first[l])

/* A single-stream state is a handle onto a private batch of one stream. */
struct DenoiseState {
  int magic;
  RNNoiseBatch *batch;
  RNNModel *owned_model; /* default model loaded on behalf of rnnoise_init(st, NULL) */
};

/* ------------------------------------------------------------------------------------------ */
static RNNModel *model_finish(RNNModel *m) {
  const void *p = m->blob ? m->blob : m->const_blob;
  if (b200_host_model_parse(&m->host, p, m->blob_len) != 0) {
    rnnoise_model_free(m);
    return NULL;
  }
  m->parsed = 1;
  return m;
}

RNNModel *rnnoise_model_from_buffer(const void *ptr, int len) {
  RNNModel *m;
  if (!ptr || len <= 0) return NULL;
  m = (RNNModel *)calloc(1, sizeof(*m));
  if (!m) return NULL;
  m->const_blob = ptr;
  m->blob_len = len;
  return model_finish(m);
}

RNNModel *rnnoise_model_from_file(FILE *f) {
  RNNModel *m;
  long len;
  if (!f) return NULL;
  if (fseek(f, 0, SEEK_END) != 0) return NULL;
  len = ftell(f);
  if (len <= 0 || fseek(f, 0, SEEK_SET) != 0) return NULL;
  m = (RNNModel *)calloc(1, sizeof(*m));
  if (!m) return NULL;
  m->blob_len = (int)len;
  m->blob = malloc((size_t)len);
  if (!m->blob || fread(m->blob, (size_t)len, 1, f) != 1) {
    rnnoise_model_free(m);
    return NULL;
  }
  return model_finish(m);
}

RNNModel *rnnoise_model_from_filename(const char *filename) {
  RNNModel *m;
  FILE *f;
  if (!filename) return NULL;
  f = fopen(filename, "rb");
  if (!f) return NULL;
  m = rnnoise_model_from_file(f); /* contents are copied, so the FILE can be closed right away */
  fclose(f);
  return m;
}

void rnnoise_model_free(RNNModel *model) {
  if (!model) return;
  if (model->parsed) b200_host_model_clear(&model->host);
  free(model->blob);
  free(model);
}

/* ------------------------------------------------------------------------------------------ */
/* Streams are independent (no cross-stream term anywhere in rnnoise_process_frame, denoise.c:457-504), so a
 * batch shards over devices as contiguous stream ranges (SURVEY 8e: stream i -> device floor(i * G / S)) with
 * no collective; each device's shard is then split into lanes as for a single device. */
RNNoiseBatch *rnnoise_batch_create_multi(RNNModel *model, int nb_streams, const int *devices, int nb_devices) {
  RNNoiseBatch *b;
  int k, s0, cnt, base, rem;
  if (!model || !model->parsed || nb_streams < 1 || !devices || nb_devices < 1 || nb_devices > B200_MAX_DEVICES) return NULL;
  if (nb_devices > nb_streams) nb_devices = nb_streams;
  for (k = 0; k < nb_devices; k++)
    if (devices[k] < 0) return NULL;
  b = (RNNoiseBatch *)calloc(1, sizeof(*b));
  if (!b) return NULL;
  b->nb_streams = nb_streams;
  b->nb_devices = nb_devices;
  base = nb_streams / nb_devices; rem = nb_streams % nb_devices;
  s0 = 0;
  for (k = 0; k < nb_devices; k++, s0 += cnt) {
    cnt = base + (k < rem ? 1 : 0);
    b->device[k] = devices[k];
    b->dev_lane[k] = k;
    b->first[k] = s0;
    b->first[k + 1] = s0 + cnt;
    b->engine[k] = b200_engine_create(&model->host, cnt, devices[k]);
    if (!b->engine[k]) {
      rnnoise_batch_destroy(b);
      return NULL;
    }
    b->lanes++;
  }
  b->dev_lane[nb_devices] = b->lanes;
  if (nb_devices > 1) {
    b->workers = (Worker *)calloc((size_t)nb_devices, sizeof(Worker));
    if (!b->workers) { rnnoise_batch_destroy(b); return NULL; }
    for (k = 0; k < nb_devices; k++) {
      Worker *w = &b->workers[k];
      w->e = b->engine[k];
      pthread_mutex_init(&w->mu, NULL);
      pthread_cond_init(&w->cv, NULL);
      if (pthread_create(&w->th, NULL, worker_main, w) != 0) {
        w->e = NULL;   /* marks "no thread" for the destructor */
        rnnoise_batch_destroy(b);
        return NULL;
      }
    }
  }
  return b;
}

RNNoiseBatch *rnnoise_batch_create(RNNModel *model, int nb_streams, int device) {
  return rnnoise_batch_create_multi(model, nb_streams, &device, 1);
}

void rnnoise_batch_destroy(RNNoiseBatch *b) {
  int l;
  if (!b) return;
  if (b->workers) {
    for (l = 0; l < b->nb_devices; l++) {
      Worker *w = &b->workers[l];
      if (!w->e) continue;
      pthread_mutex_lock(&w->mu);
      w->state = -1;
      pthread_cond_broadcast(&w->cv);
      pthread_mutex_unlock(&w->mu);
      pthread_join(w->th, NULL);
      pthread_mutex_destroy(&w->mu);
      pthread_cond_destroy(&w->cv);
    }
    free(b->workers);
    b->workers = NULL;
  }
  for (l = 0; l < B200_MAX_ENGINES; l++)
    if (b->engine[l]) b200_engine_destroy(b->engine[l]);
  free(b);
}

int rnnoise_batch_get_devices(const RNNoiseBatch *b) { return b ? b->nb_devices : 0; }
int rnnoise_batch_get_shard(const RNNoiseBatch *b, int k, int *device, int *first_stream, int *nb_streams) {
  if (!b || k < 0 || k >= b->nb_devices) return -1;
  if (device) *device = b->device[k];
  if (first_stream) *first_stream = b->first[b->dev_lane[k]];
  if (nb_streams) *nb_streams = b->first[b->dev_lane[k + 1]] - b->first[b->dev_lane[k]];
  return 0;
}

int rnnoise_batch_get_streams(const RNNoiseBatch *b) { return b ? b->nb_streams : 0; }
int rnnoise_batch_get_lanes(const RNNoiseBatch *b) { return b ? b200_engine_ranges(b->engine[0]) : 0; }

/* every per-frame entry point fans out over the lanes with the lane's offset into the caller's buffers */
#define PCM_AT(p, b, l, T, type) ((type *)(p) + (size_t)(b)->first[l] * (T) * FRAME_SIZE)
#define VAD_AT(p, b, l, T) ((p) ? (p) + (size_t)(b)->first[l] * (T) : NULL)
#define ARR_AT(p, b, l) ((p) ? (p) + (b)->first[l] : NULL)
#define FOR_LANES(b, l) for (l = 0; l < (b)->lanes; l++)

int rnnoise_batch_sync(RNNoiseBatch *b) {
  Job jobs[B200_MAX_ENGINES];
  int l;
  if (!b) return -1;
  FOR_LANES(b, l) { memset(&jobs[l], 0, sizeof(Job)); jobs[l].kind = J_SYNC; }
  return run_jobs(b, jobs);
}

/* Error discipline of the per-frame entry points: everything that can be checked is checked on EVERY lane before
 * anything is enqueued (arguments, a pending prefilter hint); such a failure returns -1 and leaves the batch as
 * it was.  A failure after that point (a CUDA error in some lane) leaves earlier lanes one frame ahead of later
 * ones, which cannot be repaired: the batch is marked poisoned and every following per-frame call returns -1;
 * destroy it.  need_idle: the entry point refuses to run across a pending rnnoise_batch_prefilter_device() hint. */
static int frame_call_ok(RNNoiseBatch *b, int need_idle, int single_device) {
  int l;
  if (!b || b->poisoned) return 0;
  if (single_device && b->nb_devices != 1) return 0;   /* one device pointer cannot address several devices */
  if (need_idle)
    FOR_LANES(b, l)
      if (b200_engine_prefilter_ahead(b->engine[l]) != 0) return 0;
  return 1;
}
#define FAN_OUT(b, l, call)          \
  do {                               \
    FOR_LANES(b, l)                  \
      if (call) {                    \
        (b)->poisoned = 1;           \
        return -1;                   \
      }                              \
  } while (0)

static int fan_out_jobs(RNNoiseBatch *b, const Job *jobs) {
  if (run_jobs(b, jobs) != 0) {
    b->poisoned = 1;
    return -1;
  }
  return 0;
}
int rnnoise_process_frame_batch_async(RNNoiseBatch *b, float *out, const float *in, float *vad) {
  Job jobs[B200_MAX_ENGINES];
  int l;
  if (!out || !in || !frame_call_ok(b, 1, 0)) return -1;
  FOR_LANES(b, l) {
    Job j = {J_HOST_ASYNC, PCM_AT(out, b, l, 1, float), PCM_AT(in, b, l, 1, const float), VAD_AT(vad, b, l, 1), 1, 0};
    jobs[l] = j;
  }
  return fan_out_jobs(b, jobs);
}
int rnnoise_process_frame_batch(RNNoiseBatch *b, float *out, const float *in, float *vad) {
  if (rnnoise_process_frame_batch_async(b, out, in, vad) != 0) return -1;
  return rnnoise_batch_sync(b);
}
int rnnoise_process_frame_batch_s16_async(RNNoiseBatch *b, short *out, const short *in, float *vad) {
  Job jobs[B200_MAX_ENGINES];
  int l;
  if (!out || !in || !frame_call_ok(b, 1, 0)) return -1;
  FOR_LANES(b, l) {
    Job j = {J_HOST_ASYNC, PCM_AT(out, b, l, 1, short), PCM_AT(in, b, l, 1, const short), VAD_AT(vad, b, l, 1), 1, 1};
    jobs[l] = j;
  }
  return fan_out_jobs(b, jobs);
}
int rnnoise_process_frame_batch_s16(RNNoiseBatch *b, short *out, const short *in, float *vad) {
  if (rnnoise_process_frame_batch_s16_async(b, out, in, vad) != 0) return -1;
  return rnnoise_batch_sync(b);
}
int rnnoise_process_frame_batch_device(RNNoiseBatch *b, float *d_out, const float *d_in, float *d_vad) {
  int l;
  if (!d_out || !d_in || !frame_call_ok(b, 0, 1)) return -1;
  FAN_OUT(b, l, b200_engine_frame_device(b->engine[l], PCM_AT(d_out, b, l, 1, float), PCM_AT(d_in, b, l, 1, const float), VAD_AT(d_vad, b, l, 1)));
  return 0;
}
int rnnoise_process_frame_batch_device_s16(RNNoiseBatch *b, short *d_out, const short *d_in, float *d_vad) {
  int l;
  if (!d_out || !d_in || !frame_call_ok(b, 0, 1)) return -1;
  FAN_OUT(b, l, b200_engine_frame_device_s16(b->engine[l], PCM_AT(d_out, b, l, 1, short), PCM_AT(d_in, b, l, 1, const short), VAD_AT(d_vad, b, l, 1)));
  return 0;
}
/* Multi-device form of the device-pointer call: d_in[k] / d_out[k] / d_vad[k] live on device k of the batch
 * (rnnoise_batch_get_shard) and hold that device's shard, [shard streams][480] / [shard streams]. */
#define DEV_OF_LANE(b, l, k) do { while ((l) >= (b)->dev_lane[(k) + 1]) (k)++; } while (0)
#define SHARD_OFF(b, l, k) ((size_t)((b)->first[l] - (b)->first[(b)->dev_lane[k]]))
int rnnoise_process_frame_batch_device_multi(RNNoiseBatch *b, float *const *d_out, const float *const *d_in, float *const *d_vad) {
  Job jobs[B200_MAX_ENGINES];
  int l, k = 0;
  if (!d_out || !d_in || !frame_call_ok(b, 0, 0)) return -1;
  for (l = 0; l < b->nb_devices; l++)
    if (!d_out[l] || !d_in[l]) return -1;
  FOR_LANES(b, l) {
    DEV_OF_LANE(b, l, k);
    {
      Job j = {J_DEVICE, d_out[k] + SHARD_OFF(b, l, k) * FRAME_SIZE, d_in[k] + SHARD_OFF(b, l, k) * FRAME_SIZE,
               d_vad && d_vad[k] ? d_vad[k] + SHARD_OFF(b, l, k) : NULL, 1, 0};
      jobs[l] = j;
    }
  }
  return fan_out_jobs(b, jobs);
}
int rnnoise_batch_prefilter_device_multi(RNNoiseBatch *b, const float *const *d_in_next) {
  Job jobs[B200_MAX_ENGINES];
  int l, k = 0;
  if (!d_in_next || !frame_call_ok(b, 0, 0)) return -1;
  for (l = 0; l < b->nb_devices; l++)
    if (!d_in_next[l]) return -1;
  FOR_LANES(b, l)
    if (b200_engine_prefilter_ahead(b->engine[l]) >= 2) return -1;
  FOR_LANES(b, l) {
    DEV_OF_LANE(b, l, k);
    {
      Job j = {J_PREFILTER, NULL, d_in_next[k] + SHARD_OFF(b, l, k) * FRAME_SIZE, NULL, 1, 0};
      jobs[l] = j;
    }
  }
  return fan_out_jobs(b, jobs);
}
static int frames_host(RNNoiseBatch *b, void *out, const void *in, float *vad, int T, int s16) {
  int l;
  if (!out || !in || T < 1 || !frame_call_ok(b, 1, 0)) return -1;
  {
    Job jobs[B200_MAX_ENGINES];
    FOR_LANES(b, l) {
      void *o = s16 ? (void *)PCM_AT(out, b, l, T, short) : (void *)PCM_AT(out, b, l, T, float);
      const void *i = s16 ? (const void *)PCM_AT(in, b, l, T, const short) : (const void *)PCM_AT(in, b, l, T, const float);
      Job j = {J_FRAMES_HOST, o, i, VAD_AT(vad, b, l, T), T, s16};
      jobs[l] = j;
    }
    if (fan_out_jobs(b, jobs) != 0) return -1;
  }
  return rnnoise_batch_sync(b);
}
int rnnoise_process_frames_batch(RNNoiseBatch *b, float *out, const float *in, float *vad, int nb_frames) {
  return frames_host(b, out, in, vad, nb_frames, 0);
}
int rnnoise_process_frames_batch_s16(RNNoiseBatch *b, short *out, const short *in, float *vad, int nb_frames) {
  return frames_host(b, out, in, vad, nb_frames, 1);
}
int rnnoise_process_frames_batch_device(RNNoiseBatch *b, float *d_out, const float *d_in, float *d_vad, int nb_frames) {
  int l;
  if (!d_out || !d_in || nb_frames < 1 || !frame_call_ok(b, 1, 1)) return -1;
  FAN_OUT(b, l, b200_engine_frames_device(b->engine[l], PCM_AT(d_out, b, l, nb_frames, float), PCM_AT(d_in, b, l, nb_frames, const float),
                                          VAD_AT(d_vad, b, l, nb_frames), nb_frames, 0));
  return 0;
}
int rnnoise_process_frames_batch_device_s16(RNNoiseBatch *b, short *d_out, const short *d_in, float *d_vad, int nb_frames) {
  int l;
  if (!d_out || !d_in || nb_frames < 1 || !frame_call_ok(b, 1, 1)) return -1;
  FAN_OUT(b, l, b200_engine_frames_device(b->engine[l], PCM_AT(d_out, b, l, nb_frames, short), PCM_AT(d_in, b, l, nb_frames, const short),
                                          VAD_AT(d_vad, b, l, nb_frames), nb_frames, 1));
  return 0;
}
int rnnoise_batch_train_features(RNNoiseBatch *b, float *rec, const float *clean, const float *noisy, const float *vad_target,
                                 const int *noise_free, const int *lowpass, const int *band_lp) {
  int l;
  if (!rec || !clean || !noisy || !frame_call_ok(b, 1, 0)) return -1;
  FAN_OUT(b, l, b200_engine_train_features_host(b->engine[l], rec + (size_t)b->first[l] * RNNOISE_TRAIN_RECORD, PCM_AT(clean, b, l, 1, const float),
                                                PCM_AT(noisy, b, l, 1, const float), ARR_AT(vad_target, b, l), ARR_AT(noise_free, b, l),
                                                ARR_AT(lowpass, b, l), ARR_AT(band_lp, b, l)));
  return 0;
}
int rnnoise_batch_train_features_device(RNNoiseBatch *b, float *d_rec, const float *d_clean, const float *d_noisy,
                                        const float *d_vad_target, const int *d_noise_free, const int *d_lowpass, const int *d_band_lp) {
  int l;
  if (!d_rec || !d_clean || !d_noisy || !frame_call_ok(b, 1, 1)) return -1;
  FAN_OUT(b, l, b200_engine_train_features_device(b->engine[l], d_rec + (size_t)b->first[l] * RNNOISE_TRAIN_RECORD, PCM_AT(d_clean, b, l, 1, const float),
                                                  PCM_AT(d_noisy, b, l, 1, const float), ARR_AT(d_vad_target, b, l), ARR_AT(d_noise_free, b, l),
                                                  ARR_AT(d_lowpass, b, l), ARR_AT(d_band_lp, b, l)));
  return 0;
}
int rnnoise_batch_timeline_read(RNNoiseBatch *b, float *ms, int capacity) {
  return b ? b200_engine_timeline_read(b->engine[0], ms, capacity) : -1;   /* first lane */
}
int rnnoise_batch_prefilter_device(RNNoiseBatch *b, const float *d_in_next) {
  int l;
  if (!d_in_next || !frame_call_ok(b, 0, 1)) return -1;
  FOR_LANES(b, l)
    if (b200_engine_prefilter_ahead(b->engine[l]) >= 2) return -1;   /* at most two frames ahead: nothing enqueued yet */
  FAN_OUT(b, l, b200_engine_prefilter_device(b->engine[l], PCM_AT(d_in_next, b, l, 1, const float)));
  return 0;
}
/* Every lane keeps its private streams (the three pipeline stages of engine.cu) and brackets each device-pointer
 * call with the caller's stream (engine.cu: parent_enter/leave): the kernels that read the caller's input or write
 * its output start after the work already enqueued on that stream, and the stream waits for the call's completion. */
int rnnoise_batch_set_stream(RNNoiseBatch *b, void *s) {
  int l;
  if (!b || b->nb_devices != 1) return -1;
  FOR_LANES(b, l)
    if (b200_engine_set_parent(b->engine[l], s)) return -1;
  return 0;
}
/* streams[k] = a cudaStream_t of device k of the batch (NULL entries / NULL array restore the private streams) */
int rnnoise_batch_set_stream_multi(RNNoiseBatch *b, void *const *streams) {
  int l, k = 0;
  if (!b) return -1;
  FOR_LANES(b, l) {
    void *s;
    DEV_OF_LANE(b, l, k);
    s = streams ? streams[k] : NULL;
    if (b200_engine_set_parent(b->engine[l], s)) return -1;
  }
  return 0;
}
int rnnoise_batch_debug_set_frame_counter(RNNoiseBatch *b, long long frames) {
  int l;
  if (!b) return -1;
  FOR_LANES(b, l)
    if (b200_engine_prefilter_ahead(b->engine[l]) != 0) return -1;
  FOR_LANES(b, l)
    if (b200_engine_debug_set_frames(b->engine[l], frames)) return -1;
  return 0;
}
static int lane_of(const RNNoiseBatch *b, int s) {
  int l;
  for (l = 0; l < b->lanes; l++)
    if (s < b->first[l + 1]) return l;
  return b->lanes - 1;
}
int rnnoise_batch_reset_stream(RNNoiseBatch *b, int s) {
  int l;
  if (!b || b->poisoned || s < 0 || s >= b->nb_streams) return -1;
  l = lane_of(b, s);
  return b200_engine_reset_stream(b->engine[l], s - b->first[l]);
}
int rnnoise_batch_launches_per_frame(const RNNoiseBatch *b) { return b ? b->lanes * b200_engine_launches_per_frame(b->engine[0]) : 0; }   /* all devices */
int rnnoise_batch_profile(RNNoiseBatch *b, int enable) {
  int l, rc = 0;
  if (!b) return -1;
  FOR_LANES(b, l) rc |= b200_engine_profile(b->engine[l], enable);
  return rc ? -1 : 0;
}
/* per-kernel times are summed over the lanes (in profiling mode the lanes run one after the other) */
int rnnoise_batch_profile_read(RNNoiseBatch *b, float *ms, const char **names, int capacity, int *frames) {
  float lane_ms[32];
  int l, i, n = 0;
  if (!b || !ms) return -1;
  FOR_LANES(b, l) {
    n = b200_engine_profile_read(b->engine[l], l == 0 ? ms : lane_ms, names, capacity < 32 ? capacity : 32, frames);
    if (n < 0) return -1;
    if (l > 0)
      for (i = 0; i < n; i++) ms[i] += lane_ms[i];
  }
  return n;
}
int rnnoise_batch_debug_read_all(RNNoiseBatch *b, int what, float *dst, int capacity) {
  int l, n = -1, per;
  if (!b || !dst || b->nb_streams < 1 || capacity % b->nb_streams) return -1;
  per = capacity / b->nb_streams; /* the caller's row length; must equal the item's length */
  FOR_LANES(b, l) {
    n = b200_engine_debug_read_all(b->engine[l], what, dst + (size_t)b->first[l] * per, LANE_COUNT(b, l) * per);
    if (n != per) return -1;
  }
  return n;
}
int rnnoise_batch_debug_read(RNNoiseBatch *b, int what, int stream, float *dst, int capacity) {
  int l;
  if (!b || stream < 0 || stream >= b->nb_streams) return -1;
  l = lane_of(b, stream);
  return b200_engine_debug_read(b->engine[l], what, stream - b->first[l], dst, capacity);
}

/* ------------------------------------------------------------------------------------------ */
int rnnoise_get_size(void) { return (int)sizeof(DenoiseState); }
int rnnoise_get_frame_size(void) { return FRAME_SIZE; }

int rnnoise_init(DenoiseState *st, RNNModel *model) {
  int device = 0;
  const char *dev;
  if (!st) return -1;
  memset(st, 0, sizeof(*st));
  if (model == NULL) {
    /* no built-in weights in this build (see rnnoise.h): fall back to the configured blob */
    const char *path = getenv("RNNOISE_B200_DEFAULT_MODEL");
    if (!path) return -1;
    st->owned_model = rnnoise_model_from_filename(path);
    if (!st->owned_model) return -1;
    model = st->owned_model;
  }
  dev = getenv("RNNOISE_B200_DEVICE");
  if (dev) device = atoi(dev);
  st->batch = rnnoise_batch_create(model, 1, device);
  if (!st->batch) {
    if (st->owned_model) rnnoise_model_free(st->owned_model);
    st->owned_model = NULL;
    return -1;
  }
  st->magic = STATE_MAGIC;
  return 0;
}

DenoiseState *rnnoise_create(RNNModel *model) {
  DenoiseState *st = (DenoiseState *)malloc(sizeof(*st));
  if (!st) return NULL;
  if (rnnoise_init(st, model) != 0) {
    free(st);
    return NULL;
  }
  return st;
}

void rnnoise_destroy_inplace(DenoiseState *st) {
  if (!st || st->magic != STATE_MAGIC) return;
  rnnoise_batch_destroy(st->batch);
  if (st->owned_model) rnnoise_model_free(st->owned_model);
  memset(st, 0, sizeof(*st));
}

void rnnoise_destroy(DenoiseState *st) {
  if (!st) return;
  rnnoise_destroy_inplace(st);
  free(st);
}

float rnnoise_process_frame(DenoiseState *st, float *out, const float *in) {
  float vad = 0.f;
  if (!st || st->magic != STATE_MAGIC) return 0.f;
  if (rnnoise_process_frame_batch(st->batch, out, in, &vad) != 0) return 0.f;
  return vad;
}
