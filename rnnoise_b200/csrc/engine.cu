// engine.cu -- device arena, model upload and the per-frame kernel sequence of the GPU engine.
//
// One frame of every stream =
//   k_biquad (thread/stream) -> k_pitch, k_spectrum (CTA/stream) -> k_conv1 -> conv2 -> GRU x3 -> k_heads
//   -> k_synthesis (CTA/stream)
// state lives in HBM between frames (layout: DESIGN.md "Data layout"); the frame index (host-side
// counter, passed to the kernels) selects the ping-pong halves and the pitch-ring base.  k_biquad
// only depends on the previous k_biquad and on the frame's input, so it runs on its own stream one
// frame ahead of the rest whenever the input is known early (pipelined host call, prefilter hint).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

// NVTX v3 is header-only: the ranges cost a relaxed load each unless a tool (nsys, ncu --nvtx) is attached.
#include <nvtx3/nvToolsExt.h>

#include "../../include/rnnoise.h"
#include "dsp_stream.cuh"
#include "dsp_pitch.cuh"
#include "dsp_tables.hpp"
#include "engine.h"
#include "rnn_kernels.cuh"
#include "gru_tc.cuh"
#include "heads_kernel.cuh"
#include "net_kernel.cuh"

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      fprintf(stderr, "[rnnoise_b200] %s failed: %s (%s:%d)\n", #call, cudaGetErrorString(e_), \
              __FILE__, __LINE__);                                                        \
      return -1;                                                                          \
    }                                                                                     \
  } while (0)

// Host-side trace ranges (SURVEY section 5 "tracing"): one per public engine call and one per pipeline stage of a frame
// (front = biquad/pitch/spectrum enqueue, network, tail = heads/synthesis), so a timeline shows the enqueue cost of
// every stage next to the kernels it launched.
struct NvtxRange {
  explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#define NVTX_SCOPE(name) NvtxRange nvtx_scope_(name)
struct NvtxStages {   // consecutive ranges inside one function; closed on every return path
  bool open = false;
  void next(const char *name) { if (open) nvtxRangePop(); nvtxRangePushA(name); open = true; }
  ~NvtxStages() { if (open) nvtxRangePop(); }
};

// ------------------------------------------------------------------------------------------------
// Per-stream state in HBM (all [S][len], stream-major so one CTA reads its stream contiguously)
// ------------------------------------------------------------------------------------------------
struct Arena {
  int S, cond, gru;
  int Kp, Kcp;         // byte row strides of the u8 operand rows: gru and 3 * cond rounded up to the 128-byte swizzle atom
                       // (the pad bytes meet zero weights in the GEMMs, so they never contribute)
  // DSP state
  float *ring;         // [S][1728] pitch history ring (analysis_mem is its newest 480 samples)
  float *synth_mem;    // [S][480]
  float *hp_mem;       // [S][2]
  float *spec;         // [3][S][2][962] X and P of frame f in slot f % 3 (f-1 is the "delayed" frame; the third
                       //                slot lets the analysis of frame f+1 overlap the synthesis of frame f)
  float *band;         // [3][S][96]     Ex, Ep, Exp, same rotation
  float *lastg;        // [S][32]
  float *pitch_state;  // [S][2] {last_period (int bits), last_gain}
  // network state
  float *conv1_state;  // [S][130]
  uint8_t *c2in;       // [S][Kcp] u8 operand row of conv2: [memory (2 frames of conv1 output) | newest | pad]
  float *hbuf;         // [2][3][S][gru] ping-pong GRU states
  uint8_t *hbuf_u8;    // [2][3][S][Kp] their u8 = 127 + rne(127 h) mirrors (tensor-core A operands)
  uint8_t *conv2_out_u8; // [S][Kp]
  // per-frame scratch
  float *xb;           // [2][S][480] high-passed input, double-buffered by frame parity
  float *features;     // [2][S][65] by frame parity (frame f+1's analysis overlaps frame f's network)
  int *silence;        // [2][S]
  float *conv2_out;    // [2][S][gru] by frame parity (the output heads of frame f run beside the network of frame f+1)
  float *gains;        // [S][32]
  float *vad;          // [S]
};

// ------------------------------------------------------------------------------------------------
// DSP kernels
// ------------------------------------------------------------------------------------------------

// High-pass biquad (rnn_biquad, denoise.c:409-419): strictly serial per stream (each step rounds
// the state to float), so one THREAD owns one stream; a warp transposes 32x32 tiles through shared
// memory so that global traffic stays coalesced.  grid = ceil(S/32), block = 32.
// `in` is float PCM, or 16-bit PCM when in_s16 != 0 (widened exactly like examples/rnnoise_demo.c:56);
// stream s starts at element s * stride (FRAME_SIZE for frame-at-a-time calls, T * FRAME_SIZE inside
// a multi-frame call whose buffers hold each stream's audio contiguously).
// Every DSP kernel works on a RANGE [r0, r1) of the batch's streams (engine.cu "ranges": the front and the tail of the
// frame pipeline run as several sub-grids on their own CUDA streams, the network over the whole batch).
__global__ void __launch_bounds__(32) k_biquad(Arena a, const void *__restrict__ in_, int frame, int in_s16, int stride, int r0, int r1) {
  const float *in = (const float *)in_;
  const short *in16 = (const short *)in_;
  __shared__ float tile[32][33];
  const int lane = threadIdx.x, s0 = r0 + blockIdx.x * 32, s = s0 + lane;
  float *xb = a.xb + (size_t)(frame & 1) * a.S * FRAME_SIZE;
  float m0 = 0.f, m1 = 0.f;
  if (s < r1) { m0 = a.hp_mem[2 * s]; m1 = a.hp_mem[2 * s + 1]; }
  const int rows = min(32, r1 - s0);
  for (int c = 0; c < FRAME_SIZE / 32; c++) {
    if (in_s16)
      for (int r = 0; r < rows; r++) tile[r][lane] = (float)in16[(size_t)(s0 + r) * stride + c * 32 + lane];
    else
      for (int r = 0; r < rows; r++) tile[r][lane] = in[(size_t)(s0 + r) * stride + c * 32 + lane];
    __syncwarp();
    if (s < r1) {
#pragma unroll 4
      for (int t = 0; t < 32; t++) tile[lane][t] = biquad_step(tile[lane][t], m0, m1);
    }
    __syncwarp();
    for (int r = 0; r < rows; r++) xb[(size_t)(s0 + r) * FRAME_SIZE + c * 32 + lane] = tile[r][lane];
    __syncwarp();
  }
  if (s < r1) { a.hp_mem[2 * s] = m0; a.hp_mem[2 * s + 1] = m1; }
}

// grid = ceil(S / PITCH_NS), block = PITCH_NS * PITCH_THREADS, dynamic smem = PITCH_NS * SM_PITCH_TOTAL floats
#ifndef PITCH_MIN_CTAS
#define PITCH_MIN_CTAS (2048 / (PITCH_NS * PITCH_THREADS) < 20 ? 2048 / (PITCH_NS * PITCH_THREADS) : 20)   // 32 regs/thread
#endif
__global__ void __launch_bounds__(PITCH_NS *PITCH_THREADS, PITCH_MIN_CTAS)
k_pitch(Arena a, const DspTables *__restrict__ T, int f, int r0, int r1) {
  extern __shared__ float sm[];
#if PITCH_NS == 1
  {
    const int s = r0 + blockIdx.x;
    PitchArgs g;   // in registers: pointers keep their (global) address space
    g.ring_base = (int)(((long long)(f + 1) * FRAME_SIZE) % PITCH_BUF_SIZE);
    g.xb = a.xb + ((size_t)(f & 1) * a.S + s) * FRAME_SIZE;
    g.ring = a.ring + (size_t)s * PITCH_BUF_SIZE;
    g.pitch_state = a.pitch_state + 2 * (size_t)s;
    pitch_streams(sm, &g, T);
  }
#else
  __shared__ PitchArgs pa[PITCH_NS];
  {
    const int grp = blockIdx.x;
    if (threadIdx.x < PITCH_NS) {
      const int s = r0 + grp * PITCH_NS + threadIdx.x;
      PitchArgs g;
      g.ring = nullptr; g.xb = nullptr; g.pitch_state = nullptr;
      g.ring_base = (int)(((long long)(f + 1) * FRAME_SIZE) % PITCH_BUF_SIZE);
      if (s < r1) {
        g.xb = a.xb + ((size_t)(f & 1) * a.S + s) * FRAME_SIZE;
        g.ring = a.ring + (size_t)s * PITCH_BUF_SIZE;
        g.pitch_state = a.pitch_state + 2 * (size_t)s;
      }
      pa[threadIdx.x] = g;
    }
    __syncthreads();
    pitch_streams(sm, pa, T);
  }
#endif
}

// Default pitch kernel (dsp_pitch.cuh): CTA = PG streams, one home warp per stream + three chain warps.
// grid = ceil(S / PG), block = PG_THREADS, dynamic smem = PG * P2_STRIDE floats
#define PITCH2_SMEM_BYTES (PG * P2_STRIDE * (int)sizeof(float))
__global__ void __launch_bounds__(PG_THREADS, PG <= 8 ? 2 : 1) k_pitch2(Arena a, int f, int r0, int r1) {
  extern __shared__ float sm[];
  const int s0 = r0 + blockIdx.x * PG;
  PitchGroup g;
  g.n = min(PG, r1 - s0);
  g.ring_base = (int)(((long long)(f + 1) * FRAME_SIZE) % PITCH_BUF_SIZE);
  g.xb = a.xb + ((size_t)(f & 1) * a.S + s0) * FRAME_SIZE;
  g.ring = a.ring + (size_t)s0 * PITCH_BUF_SIZE;
  g.pitch_state = a.pitch_state + 2 * (size_t)s0;
  pitch_group(sm, g);
}

// 12 CTAs per SM = 40 registers per thread without spills.  The shared-memory plan would admit 14, but 32 registers
// spill in the radix-5 stage.
#ifndef SPEC_MIN_BLOCKS
#define SPEC_MIN_BLOCKS 12
#endif
__global__ void __launch_bounds__(DSP_THREADS, SPEC_MIN_BLOCKS) k_spectrum(Arena a, const DspTables *__restrict__ T, int f, int r0) {
  extern __shared__ float sm[];
  const int par = f & 1, slot = f % 3;
  const int s = r0 + blockIdx.x;
  SpectrumArgs g;
  g.ring = a.ring + (size_t)s * PITCH_BUF_SIZE;
  g.ring_base = (int)(((long long)(f + 1) * FRAME_SIZE) % PITCH_BUF_SIZE);
  g.pitch_state = a.pitch_state + 2 * (size_t)s;
  g.spec_out = a.spec + ((size_t)slot * a.S + s) * (4 * FREQ_SIZE);
  g.band_out = a.band + ((size_t)slot * a.S + s) * 96;
  g.features = a.features + ((size_t)par * a.S + s) * NB_FEATURES;
  g.silence = a.silence + (size_t)par * a.S + s;
  g.lowpass = FREQ_SIZE;
  spectrum_stream<false>(sm, g, T);
}

// Training-feature extraction (src/dump_features.c:466-491): spectrum_stream<true> of the noisy frame +
// clean-frame analysis + ideal gains; one 98-float record per stream.  Per-stream arrays may be null
// (vad target 0, noise present, no low-pass).  grid = S, block = 128, dynamic smem = SM_SPEC_TOTAL floats
struct TrainIo {
  const float *clean;       // [S][480]
  float *clean_mem;         // [S][480]
  float *rec;               // [S][98]
  const float *vad_target;  // [S] or null
  const int *noise_free, *lowpass, *band_lp;   // [S] or null
};
__global__ void __launch_bounds__(DSP_THREADS) k_train_features(Arena a, const DspTables *__restrict__ T, int f, TrainIo io) {
  extern __shared__ float sm[];
  const int par = f & 1, slot = f % 3;
  const int s = blockIdx.x;
  SpectrumArgs g;
  g.ring = a.ring + (size_t)s * PITCH_BUF_SIZE;
  g.ring_base = (int)(((long long)(f + 1) * FRAME_SIZE) % PITCH_BUF_SIZE);
  g.pitch_state = a.pitch_state + 2 * (size_t)s;
  g.spec_out = a.spec + ((size_t)slot * a.S + s) * (4 * FREQ_SIZE);
  g.band_out = a.band + ((size_t)slot * a.S + s) * 96;
  g.features = io.rec + (size_t)s * TRAIN_RECORD;
  g.silence = a.silence + (size_t)par * a.S + s;
  g.lowpass = io.lowpass ? io.lowpass[s] : FREQ_SIZE;
  spectrum_stream<true>(sm, g, T);
  TrainArgs t;
  t.clean = io.clean + (size_t)s * FRAME_SIZE;
  t.clean_mem = io.clean_mem + (size_t)s * FRAME_SIZE;
  t.rec = io.rec + (size_t)s * TRAIN_RECORD;
  t.quiet = g.silence;
  t.lowpass = g.lowpass;
  t.band_lp = io.band_lp ? io.band_lp[s] : NB_BANDS;
  t.vad_target = io.vad_target ? io.vad_target[s] : 0.f;
  t.noise_free = io.noise_free ? io.noise_free[s] : 0;
  train_targets_stream(sm, t, T);
}

__global__ void __launch_bounds__(DSP_THREADS, 14) k_synthesis(Arena a, const DspTables *__restrict__ T,
                                                           void *__restrict__ out, int f, int out_s16, int stride, int r0) {
  extern __shared__ float sm[];
  const int s = r0 + blockIdx.x;
  pdl_wait();   // gains of this frame (k_heads)
  const int par = f & 1, slot = f % 3, dslot = (f + 2) % 3;   // dslot = (f - 1) mod 3
  SynthesisArgs g;
  g.spec_delayed = a.spec + ((size_t)dslot * a.S + s) * (4 * FREQ_SIZE);
  g.band_delayed = a.band + ((size_t)dslot * a.S + s) * 96;
  g.band_cur = a.band + ((size_t)slot * a.S + s) * 96;
  g.gains = a.gains + (size_t)s * NB_BANDS;
  g.silence = a.silence + (size_t)par * a.S + s;
  g.lastg = a.lastg + (size_t)s * NB_BANDS;
  g.synthesis_mem = a.synth_mem + (size_t)s * FRAME_SIZE;
  g.out = out_s16 ? nullptr : (float *)out + (size_t)s * stride;
  g.out_s16 = out_s16 ? (short *)out + (size_t)s * stride : nullptr;
  synthesis_stream(sm, g, T);
}

// ------------------------------------------------------------------------------------------------
#define NKERNELS 10
#define B200_MAX_RANGES 4
struct B200Engine {
  int device;
  Arena a;
  DevModel dm;
  DspTables *d_tables;
  cudaStream_t own_stream, stream;
  long long frames;                 // host mirror of the device frame counter
  std::vector<void *> allocs;
  // host-buffer calls: double-buffered device staging, copy streams and the events that chain
  // H2D(n) -> compute(n) -> D2H(n) while protecting slot reuse two frames later
  float *stage_in[2], *stage_out[2], *stage_vad[2];
  cudaStream_t s_h2d, s_d2h;
  // Ranges ("lanes"): the DSP stages of a frame -- analysis front (biquad -> pitch -> spectrum) and tail (output heads ->
  // synthesis) -- run as 1..4 sub-grids over contiguous stream ranges, each on its own CUDA streams, so that kernels of
  // about one wave overlap with each other and with the other pipeline stages; the network kernels, whose CTAs are
  // latency-bound whatever the grid size, run ONCE over the whole batch on `stream`.
  int nr;
  struct Range {
    int r0, r1;                      // streams [r0, r1)
    cudaStream_t s_bq, s_front, s_tail;
    cudaEvent_t ev_bq[2], ev_ana[2]; // biquad of frame f done / pitch of frame f done (xb slot free), by frame parity
    cudaEvent_t ev_front[2], ev_back[2];   // analysis of frame f done / tail (heads + synthesis) of frame f done
  } rg[B200_MAX_RANGES];
  cudaEvent_t ev_net[2];             // network of frame f done (by parity): the tails may start
  int tail_overlap;                  // 0: heads + synthesis stay on the network's stream ($RNNOISE_B200_TAIL_OVERLAP=0)
  cudaEvent_t ev_in;                 // input readiness on the caller's stream (non-prefiltered frames)
  // lanes (rnnoise_api.c splits a batch into sub-batches that run concurrently): a lane other than the
  // first keeps its own stream but orders every call after `parent` (the caller's stream) and makes
  // `parent` wait for the call's completion, so the caller sees one stream's semantics
  cudaStream_t parent;
  cudaEvent_t ev_pin, ev_pout;
  int io_stride, vad_stride;         // element strides between streams in the caller's PCM / VAD buffers
  // multi-frame host calls: double-buffered chunk staging ([S][chunk*480] in, out; [S][chunk] vad)
  void *multi_in[2], *multi_out[2];
  float *multi_vad[2];
  int multi_chunk;                   // frames per staged chunk (RNNOISE_B200_MULTI_CHUNK, default 16)
  size_t multi_bytes;                // bytes allocated per PCM staging buffer
  cudaEvent_t ev_mh2d[2], ev_mcomp[2], ev_md2h[2];
  // training-feature extraction: clean-speech analysis memory and host-call staging (allocated on first use)
  float *train_clean_mem, *train_stage;   // [S][480]; [S][2*480 + 98 + 4]
  int overlap;                       // 0: everything on one stream (RNNOISE_B200_OVERLAP=0, profiling)
  int pdl;                           // programmatic dependent launch along the network chain (RNNOISE_B200_PDL=1 enables)
  cudaEvent_t ev_h2d[2], ev_d2h[2];
  long long host_frames;
  long long bq_frames;               // frames whose high-pass prefilter has been issued
  int use_tc;                       // GRU kernel: 2 = k_tc2<true> (default), 1 = k_gru_tc, 0 = dp4a cross-check
  int conv2_tc;                     // conv2 kernel: 1 = k_tc2<false> (default), 0 = dp4a cross-check
  int pitch2;                       // pitch kernel: 1 = k_pitch2 (default), 0 = k_pitch (RNNOISE_B200_PITCH_KERNEL=v1 cross-check)
  int heads_ns;                     // k_heads2<NS, NW> tile: 1 = <1,4> 8 streams per CTA, 2 = <2,4> 16, 4 = <4,4> 32, 8 = <2,8> 32 streams on
                                    // 8 compute warps ($RNNOISE_B200_HEADS_TILE = 8 | 16 | 32 | 32w)
  int heads2;                       // heads kernel: 1 = k_heads2 (default), 0 = k_heads (RNNOISE_B200_HEADS_KERNEL=cpasync)
  GruTcMaps tc_maps[2][3];          // [frame parity][layer]
  GruTcMaps conv_maps;              // x = c2in, wi = conv2 weights
  int net_cluster;                  // CTAs per cluster of k_net: 4 (default) or 8 ($RNNOISE_B200_NET_CLUSTER; needs gru % 128 == 0)
  int net_conv1;                    // 1 = conv1 runs as k_net's prologue (default with net_fused); 0 = k_conv1 launch
  int net_fused;                    // 1 = k_net: conv2 + 3 GRU layers in one cluster kernel (default); 0 = one launch per layer
  NetMaps net_maps[2];              // [frame parity]
  NetPtrs net_ptrs[2];
  // optional per-kernel timing (rnnoise_batch_profile)
  int profiling, prof_frames;
  cudaEvent_t ev[NKERNELS + 1];
  double prof_ms[NKERNELS];
  // optional pipeline timeline ($RNNOISE_B200_TIMELINE = frames to record): timing events at the stage
  // boundaries of the first frames, on the streams the stages run on (rnnoise_batch_timeline_read)
  int tl_frames;
  std::vector<cudaEvent_t> tl;
};
enum { TL_H2D_START, TL_H2D_END, TL_BQ_END, TL_PITCH_END, TL_FRONT_END, TL_BACK_START, TL_BACK_END, TL_D2H_END, TL_POINTS };
#define TL(e, frame, point, stream) \
  do { if ((frame) < (long long)(e)->tl_frames) cudaEventRecord((e)->tl[(size_t)(frame) * TL_POINTS + (point)], (stream)); } while (0)
static const char *const kKernelNames[NKERNELS] = {"k_biquad", "k_pitch", "k_spectrum", "k_conv1", "k_conv2", "k_gru[0]",
                                                   "k_gru[1]", "k_gru[2]", "k_heads", "k_synthesis"};

// The kernels derive three things from the frame index they are handed: the ping-pong parity f & 1, the
// spectrum slot f % 3 and the pitch-ring base ((f + 1) * 480) % 1728, which has period 18 in f.  The 64-bit
// host counter is therefore reduced modulo a multiple of lcm(2, 3, 18) = 18 that fits an int: all three stay
// continuous for ever (a plain power-of-two mask would make the slot and the ring base jump at the wrap).
#define FRAME_WRAP (18LL << 24)
static inline int frame_arg(long long f) { return (int)(f % FRAME_WRAP); }

template <typename T>
static T *dalloc(B200Engine *e, size_t n, bool zero = true) {
  void *p = nullptr;
  if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) return nullptr;
  e->allocs.push_back(p);   // owned from here on: freed by b200_engine_destroy even when the memset below fails
  if (zero && cudaMemset(p, 0, n * sizeof(T)) != cudaSuccess) return nullptr;
  return (T *)p;
}
template <typename T>
static const T *upload(B200Engine *e, const T *h, size_t n) {
  T *d = dalloc<T>(e, n, false);
  if (!d) return nullptr;
  if (cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  return d;
}

// dense s8 [out][in] -> packed [in/4][out] int32 (4 consecutive inputs of one output per word)
static const int *upload_packed(B200Engine *e, const B200Layer *l) {
  const int K4 = l->nb_in / 4, N = l->nb_out;
  std::vector<int> p((size_t)K4 * N);
  for (int k4 = 0; k4 < K4; k4++)
    for (int o = 0; o < N; o++) {
      const signed char *w = l->w8 + (size_t)o * l->nb_in + 4 * k4;
      unsigned v = (unsigned)(unsigned char)w[0] | ((unsigned)(unsigned char)w[1] << 8) |
                   ((unsigned)(unsigned char)w[2] << 16) | ((unsigned)(unsigned char)w[3] << 24);
      p[(size_t)k4 * N + o] = (int)v;
    }
  return upload<int>(e, p.data(), p.size());
}
static int upload_q(B200Engine *e, DevLayerQ *d, const B200Layer *l) {
  d->wp = upload_packed(e, l);
  d->scale = upload<float>(e, l->scale, l->nb_out);
  d->subias = upload<float>(e, l->subias, l->nb_out);
  d->diag = l->diag ? upload<float>(e, l->diag, l->nb_out) : nullptr;
  d->packed = nullptr;
  return (d->wp && d->scale && d->subias && (!l->diag || d->diag)) ? 0 : -1;
}
// epilogue parameter records of one GRU layer (DevLayerQ::packed), from the host copies of its two matrices
static int upload_gru_params(B200Engine *e, DevLayerQ *rec, const B200Layer *li, const B200Layer *lr, int gru) {
  std::vector<float> p((size_t)gru * 16, 0.f);
  for (int u = 0; u < gru; u++)
    for (int g = 0; g < 3; g++) {
      float *q = &p[(size_t)u * 16 + 4 * g];
      q[0] = li->scale[g * gru + u]; q[1] = li->subias[g * gru + u];
      q[2] = lr->scale[g * gru + u]; q[3] = lr->subias[g * gru + u];
      p[(size_t)u * 16 + 12 + g] = lr->diag[g * gru + u];
    }
  rec->packed = upload<float>(e, p.data(), p.size());
  return rec->packed ? 0 : -1;
}
static int upload_f(B200Engine *e, DevLayerF *d, const B200Layer *l) {
  d->w = upload<float>(e, l->wf, (size_t)l->nb_in * l->nb_out);
  d->bias = upload<float>(e, l->bias, l->nb_out);
  return (d->w && d->bias) ? 0 : -1;
}


// ------------------------------------------------------------------------------------------------
// TMA tensor maps for the tensor-core GRU (gru_tc.cuh).  cuTensorMapEncodeTiled is fetched through
// the runtime (no link-time dependency on libcuda).
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// row-major bytes [rows][K], box = [box_rows][128 B], 128B swizzle
static int make_map_u8(CUtensorMap *m, const void *base, uint64_t rows, uint64_t K, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {K, rows};
  cuuint64_t strides[1] = {K};
  cuuint32_t box[2] = {TC_KATOM, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}
// dense s8 [3*gru][K] (rows = z|r|n outputs) -> [gru/32 slices][3 gates][32 units][K]: the 96 B-operand
// rows of one unit slice become contiguous
// K is padded with zero weights up to Kp bytes per row.
static const signed char *upload_permuted(B200Engine *e, const B200Layer *l, int gru, int units, int Kp) {
  const int K = l->nb_in;
  std::vector<signed char> p((size_t)3 * gru * Kp, 0);
  for (int sl = 0; sl < gru / units; sl++)
    for (int g = 0; g < 3; g++)
      for (int u = 0; u < units; u++)
        memcpy(&p[(((size_t)sl * 3 + g) * units + u) * Kp], l->w8 + (size_t)(g * gru + sl * units + u) * K, K);
  return upload<signed char>(e, p.data(), p.size());
}
static const signed char *upload_padded_rows(B200Engine *e, const signed char *w, int rows, int K, int Kp) {
  std::vector<signed char> p((size_t)rows * Kp, 0);
  for (int r = 0; r < rows; r++) memcpy(&p[(size_t)r * Kp], w + (size_t)r * K, K);
  return upload<signed char>(e, p.data(), p.size());
}

extern "C" void b200_engine_destroy(B200Engine *e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->own_stream) { cudaStreamSynchronize(e->own_stream); cudaStreamDestroy(e->own_stream); }
  for (int i = 0; i <= NKERNELS; i++) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
  if (e->s_h2d) { cudaStreamSynchronize(e->s_h2d); cudaStreamDestroy(e->s_h2d); }
  if (e->s_d2h) { cudaStreamSynchronize(e->s_d2h); cudaStreamDestroy(e->s_d2h); }
  for (int r = 0; r < B200_MAX_RANGES; r++) {
    B200Engine::Range &R = e->rg[r];
    if (R.s_bq) { cudaStreamSynchronize(R.s_bq); cudaStreamDestroy(R.s_bq); }
    if (R.s_front) { cudaStreamSynchronize(R.s_front); cudaStreamDestroy(R.s_front); }
    if (R.s_tail) { cudaStreamSynchronize(R.s_tail); cudaStreamDestroy(R.s_tail); }
    for (int i = 0; i < 2; i++) {
      if (R.ev_bq[i]) cudaEventDestroy(R.ev_bq[i]);
      if (R.ev_ana[i]) cudaEventDestroy(R.ev_ana[i]);
      if (R.ev_front[i]) cudaEventDestroy(R.ev_front[i]);
      if (R.ev_back[i]) cudaEventDestroy(R.ev_back[i]);
    }
  }
  if (e->ev_in) cudaEventDestroy(e->ev_in);
  if (e->ev_pin) cudaEventDestroy(e->ev_pin);
  if (e->ev_pout) cudaEventDestroy(e->ev_pout);
  for (int i = 0; i < 2; i++) {
    if (e->ev_h2d[i]) cudaEventDestroy(e->ev_h2d[i]);
    if (e->ev_d2h[i]) cudaEventDestroy(e->ev_d2h[i]);
    if (e->ev_net[i]) cudaEventDestroy(e->ev_net[i]);
    if (e->ev_mh2d[i]) cudaEventDestroy(e->ev_mh2d[i]);
    if (e->ev_mcomp[i]) cudaEventDestroy(e->ev_mcomp[i]);
    if (e->ev_md2h[i]) cudaEventDestroy(e->ev_md2h[i]);
    cudaFree(e->multi_in[i]); cudaFree(e->multi_out[i]); cudaFree(e->multi_vad[i]);
  }
  for (auto ev : e->tl) if (ev) cudaEventDestroy(ev);
  for (void *p : e->allocs) cudaFree(p);
  delete e;
}

extern "C" B200Engine *b200_engine_create(const B200HostModel *m, int S, int device) { return b200_engine_create_on(m, S, device, S); }
// device_streams = streams of the whole batch that live on this device (all lanes): the kernel choices that depend on
// how full the GPU is are made on that figure, not on the lane's share.
extern "C" B200Engine *b200_engine_create_on(const B200HostModel *m, int S, int device, int device_streams) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    fprintf(stderr, "[rnnoise_b200] no CUDA device available -- this library has no CPU path\n");
    return nullptr;
  }
  if (!m || S < 1 || device < 0 || device >= ndev) return nullptr;
  // gru: a CTA of the tensor-core kernels owns gru / 4 units in slices of 16, the heads stream 64-input chunks that
  // must not straddle two layers; cond: one conv1 output per thread of a 128-thread CTA.  The contraction lengths
  // themselves (gru, 3 * cond) are free: rows are padded to the 128-byte swizzle atom with zero weights.
  if (m->gru % 64 || m->cond % 4 || m->gru > 1024 || m->cond > 128 || m->gru < 64 || m->cond < 4) {
    fprintf(stderr, "[rnnoise_b200] unsupported model dims cond=%d gru=%d (need gru %% 64 == 0, gru <= 1024, cond %% 4 == 0, cond <= 128)\n", m->cond, m->gru);
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) return nullptr;
  B200Engine *e = new B200Engine();
  e->device = device;
  e->frames = 0;
  e->own_stream = nullptr;
  e->profiling = 0; e->prof_frames = 0;
  for (int i = 0; i <= NKERNELS; i++) e->ev[i] = nullptr;
  {
    // the engine's own stream (network + synthesis) runs at the highest priority and the analysis front at
    // the lowest (s_front below): the back half of frame f gets SM slots before the front of frame f+1
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (cudaStreamCreateWithPriority(&e->own_stream, cudaStreamNonBlocking, hi) != cudaSuccess) { delete e; return nullptr; }
  }
  e->stream = e->own_stream;
  Arena &a = e->a;
  a.S = S; a.cond = m->cond; a.gru = m->gru;
  a.Kp = (m->gru + TC_KATOM - 1) / TC_KATOM * TC_KATOM;
  a.Kcp = (3 * m->cond + TC_KATOM - 1) / TC_KATOM * TC_KATOM;
  const size_t Ss = (size_t)S;
  bool ok = true;
  ok &= !!(a.ring = dalloc<float>(e, Ss * PITCH_BUF_SIZE));
  ok &= !!(a.synth_mem = dalloc<float>(e, Ss * FRAME_SIZE));
  ok &= !!(a.hp_mem = dalloc<float>(e, Ss * 2));
  ok &= !!(a.spec = dalloc<float>(e, 3 * Ss * 4 * FREQ_SIZE));
  ok &= !!(a.band = dalloc<float>(e, 3 * Ss * 96));
  ok &= !!(a.lastg = dalloc<float>(e, Ss * NB_BANDS));
  ok &= !!(a.pitch_state = dalloc<float>(e, Ss * 2));
  ok &= !!(a.conv1_state = dalloc<float>(e, Ss * 2 * NB_FEATURES));
  ok &= !!(a.c2in = dalloc<uint8_t>(e, Ss * a.Kcp));
  if (ok) ok = cudaMemset(a.c2in, 127, Ss * a.Kcp) == cudaSuccess;   // u8 image of zeros
  ok &= !!(a.hbuf = dalloc<float>(e, 2 * 3 * Ss * m->gru));
  ok &= !!(a.hbuf_u8 = dalloc<uint8_t>(e, 2 * 3 * Ss * a.Kp));
  ok &= !!(a.conv2_out_u8 = dalloc<uint8_t>(e, Ss * a.Kp));
  if (ok) ok = cudaMemset(a.hbuf_u8, 127, 2 * 3 * Ss * a.Kp) == cudaSuccess;   // u8 image of h = 0
  if (ok) ok = cudaMemset(a.conv2_out_u8, 127, Ss * a.Kp) == cudaSuccess;
  ok &= !!(a.xb = dalloc<float>(e, 2 * Ss * FRAME_SIZE));
  ok &= !!(a.features = dalloc<float>(e, 2 * Ss * NB_FEATURES));
  ok &= !!(a.silence = dalloc<int>(e, 2 * Ss));
  ok &= !!(a.conv2_out = dalloc<float>(e, 2 * Ss * m->gru));
  ok &= !!(a.gains = dalloc<float>(e, Ss * NB_BANDS));
  ok &= !!(a.vad = dalloc<float>(e, Ss));
  e->host_frames = 0;
  e->bq_frames = 0;
  {
    const char *tl = getenv("RNNOISE_B200_TIMELINE");
    e->tl_frames = tl && atoi(tl) > 0 ? atoi(tl) : 0;
    e->tl.assign((size_t)e->tl_frames * TL_POINTS, nullptr);
    for (auto &ev : e->tl) ok &= cudaEventCreate(&ev) == cudaSuccess;
  }
  e->parent = nullptr;
  e->ev_pin = e->ev_pout = nullptr;
  ok &= cudaEventCreateWithFlags(&e->ev_pin, cudaEventDisableTiming) == cudaSuccess;
  ok &= cudaEventCreateWithFlags(&e->ev_pout, cudaEventDisableTiming) == cudaSuccess;
  e->io_stride = FRAME_SIZE;
  e->vad_stride = 1;
  e->train_clean_mem = e->train_stage = nullptr;
  e->multi_bytes = 0;
  {
    const char *mc = getenv("RNNOISE_B200_MULTI_CHUNK");
    e->multi_chunk = mc && atoi(mc) > 0 ? atoi(mc) : 16;
  }
  for (int i = 0; i < 2; i++) {
    e->multi_in[i] = e->multi_out[i] = nullptr; e->multi_vad[i] = nullptr;
    e->ev_mh2d[i] = e->ev_mcomp[i] = e->ev_md2h[i] = nullptr;
  }
  e->s_h2d = e->s_d2h = nullptr;
  memset(e->rg, 0, sizeof(e->rg));
  { const char *to = getenv("RNNOISE_B200_TAIL_OVERLAP"); e->tail_overlap = !(to && !strcmp(to, "0")); }
  e->ev_in = nullptr;
  const char *ov = getenv("RNNOISE_B200_OVERLAP");
  e->overlap = !(ov && !strcmp(ov, "0"));
  // programmatic dependent launch is opt-in: early-launched dependents hold smem/thread slots the overlapping analysis
  // kernels could use
  { const char *pd = getenv("RNNOISE_B200_PDL"); e->pdl = pd && !strcmp(pd, "1"); }
  {
    // Ranges of the DSP stages: two from 1024 to 32767 streams, else one (kernels of about one wave overlap with each
    // other and with the other stages); whole 128-stream tiles except the last.  $RNNOISE_B200_LANES overrides.
    const char *ln = getenv("RNNOISE_B200_LANES");
    int nr = ln && atoi(ln) > 0 ? atoi(ln) : (S >= 1024 && S < 32768) ? 2 : 1;
    if (nr > B200_MAX_RANGES) nr = B200_MAX_RANGES;
    while (nr > 1 && S / nr < 128) nr--;
    const int per = ((S + nr - 1) / nr + 127) / 128 * 128;
    e->nr = 0;
    for (int r = 0; r < nr && r * per < S; r++) {
      e->rg[r].r0 = r * per;
      e->rg[r].r1 = (r + 1) * per < S ? (r + 1) * per : S;
      e->nr++;
    }
    // stream priorities: the tails (oldest frame) and the network first, the analysis fronts last -- the front of frame
    // f+1 only fills what the back of frame f leaves free.  (Capping the front kernels' grid to leave room was measured
    // to be worse than the plain one-CTA-per-stream grid.)
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);   // lo = lowest priority (largest value)
    const char *pr = getenv("RNNOISE_B200_FRONT_PRIORITY");
    for (int r = 0; r < e->nr; r++) {
      B200Engine::Range &R = e->rg[r];
      ok &= cudaStreamCreateWithPriority(&R.s_tail, cudaStreamNonBlocking, hi) == cudaSuccess;
      ok &= cudaStreamCreateWithPriority(&R.s_front, cudaStreamNonBlocking, pr && !strcmp(pr, "high") ? hi : lo) == cudaSuccess;
      ok &= cudaStreamCreateWithFlags(&R.s_bq, cudaStreamNonBlocking) == cudaSuccess;
      for (int i = 0; i < 2; i++) {
        ok &= cudaEventCreateWithFlags(&R.ev_bq[i], cudaEventDisableTiming) == cudaSuccess;
        ok &= cudaEventCreateWithFlags(&R.ev_ana[i], cudaEventDisableTiming) == cudaSuccess;
        ok &= cudaEventCreateWithFlags(&R.ev_front[i], cudaEventDisableTiming) == cudaSuccess;
        ok &= cudaEventCreateWithFlags(&R.ev_back[i], cudaEventDisableTiming) == cudaSuccess;
      }
    }
  }
  ok &= cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming) == cudaSuccess;
  ok &= cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking) == cudaSuccess;
  ok &= cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; i < 2; i++) {
    ok &= !!(e->stage_in[i] = dalloc<float>(e, Ss * FRAME_SIZE));
    ok &= !!(e->stage_out[i] = dalloc<float>(e, Ss * FRAME_SIZE));
    ok &= !!(e->stage_vad[i] = dalloc<float>(e, Ss));
    e->ev_h2d[i] = e->ev_d2h[i] = e->ev_net[i] = nullptr;
    ok &= cudaEventCreateWithFlags(&e->ev_net[i], cudaEventDisableTiming) == cudaSuccess;
    ok &= cudaEventCreateWithFlags(&e->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess;
    ok &= cudaEventCreateWithFlags(&e->ev_d2h[i], cudaEventDisableTiming) == cudaSuccess;
    ok &= cudaEventCreateWithFlags(&e->ev_mh2d[i], cudaEventDisableTiming) == cudaSuccess;
    ok &= cudaEventCreateWithFlags(&e->ev_mcomp[i], cudaEventDisableTiming) == cudaSuccess;
    ok &= cudaEventCreateWithFlags(&e->ev_md2h[i], cudaEventDisableTiming) == cudaSuccess;
  }
  DspTables *ht = new DspTables();
  b200_fill_dsp_tables(ht);
  e->d_tables = (DspTables *)upload<DspTables>(e, ht, 1);
  delete ht;
  ok &= !!e->d_tables;
  DevModel &dm = e->dm;
  dm.cond = m->cond; dm.gru = m->gru;
  ok = ok && upload_f(e, &dm.conv1, &m->conv1) == 0 && upload_f(e, &dm.dense_out, &m->dense_out) == 0 &&
       upload_f(e, &dm.vad_dense, &m->vad_dense) == 0 && upload_q(e, &dm.conv2, &m->conv2) == 0;
  for (int k = 0; k < 3 && ok; k++)
    ok = upload_q(e, &dm.gru_in[k], &m->gru_in[k]) == 0 && upload_q(e, &dm.gru_rec[k], &m->gru_rec[k]) == 0 &&
         m->gru_rec[k].diag && upload_gru_params(e, &dm.gru_rec[k], &m->gru_in[k], &m->gru_rec[k], m->gru) == 0;
  // tensor-core GRU path: permuted weights + TMA maps for both frame parities
  // RNNOISE_B200_GRU_KERNEL = tc2 (default: persistent pipelined wgmma) | tc1 (one tile per CTA) |
  // dp4a (CUDA-core cross-check); all three produce identical bits
  { const char *hk = getenv("RNNOISE_B200_HEADS_KERNEL"); e->heads2 = !(hk && !strcmp(hk, "cpasync")); }
  // Pitch kernel: v1 (4 streams x 96 threads per CTA, 20 streams resident per SM) is the default; v2 (k_pitch2, 16
  // streams per CTA, far fewer instructions but one CTA per SM) has the same throughput per SM and only wins when a
  // lane is exactly one wave of its CTAs; $RNNOISE_B200_PITCH_KERNEL = v1 | v2.
  { const char *pk = getenv("RNNOISE_B200_PITCH_KERNEL"); e->pitch2 = pk && !strcmp(pk, "v2"); }
  ok = ok && cudaFuncSetAttribute(k_pitch2, cudaFuncAttributeMaxDynamicSharedMemorySize, PITCH2_SMEM_BYTES) == cudaSuccess;
  // streams per CTA of the heads kernel: 16 while the batch is small (twice the CTAs: lower latency), 32 once the GPU is
  // full (fewer, fatter CTAs disturb the other stages less)
  { const char *ht = getenv("RNNOISE_B200_HEADS_TILE"); e->heads_ns = ht ? (!strcmp(ht, "32w") ? 8 : !strcmp(ht, "32") ? 4 : !strcmp(ht, "8") ? 1 : 2) : device_streams >= 4096 ? 4 : 2; }
  ok = ok && cudaFuncSetAttribute(k_heads2<1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, h2_smem_bytes<1>()) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(k_heads2<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, h2_smem_bytes<4>()) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(k_heads2<2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, h2_smem_bytes<2>()) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(k_heads2<2, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, h2_smem_bytes<2, 8>()) == cudaSuccess;
  const char *gk = getenv("RNNOISE_B200_GRU_KERNEL");
  e->use_tc = gk && !strcmp(gk, "dp4a") ? 0 : gk && !strcmp(gk, "tc1") && m->gru % 128 == 0 ? 1 : 2;
  if (ok && e->use_tc) {
    const size_t hs = Ss * a.Kp;
    const int units = e->use_tc == 1 ? TC_UNITS : P_SLICE;
    for (int l = 0; l < 3 && ok; l++) {
      const signed char *wi = upload_permuted(e, &m->gru_in[l], m->gru, units, a.Kp), *wr = upload_permuted(e, &m->gru_rec[l], m->gru, units, a.Kp);
      ok = wi && wr;
      for (int par = 0; par < 2 && ok; par++) {
        GruTcMaps &mp = e->tc_maps[par][l];
        const uint8_t *x = l == 0 ? a.conv2_out_u8 : a.hbuf_u8 + ((size_t)par * 3 + l - 1) * hs;
        const uint8_t *h = a.hbuf_u8 + ((size_t)(par ^ 1) * 3 + l) * hs;
        ok = make_map_u8(&mp.x, x, S, a.Kp, TC_M) == 0 && make_map_u8(&mp.h, h, S, a.Kp, TC_M) == 0 &&
             make_map_u8(&mp.wi, wi, 3 * m->gru, a.Kp, 3 * units) == 0 && make_map_u8(&mp.wr, wr, 3 * m->gru, a.Kp, 3 * units) == 0;
      }
    }
    ok = ok && cudaFuncSetAttribute(k_gru_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, gru_tc_smem_bytes(m->gru)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(k_tc2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2_smem_bytes<true>(a.Kp, m->gru)) == cudaSuccess;
    if (!ok) fprintf(stderr, "[rnnoise_b200] tensor-core GRU setup failed\n");
  }
  // conv2 on the tensor cores: K = 3 * cond padded to whole 128-byte swizzle atoms
  const char *ck = getenv("RNNOISE_B200_CONV2_KERNEL");
  e->conv2_tc = !(ck && !strcmp(ck, "dp4a"));
  if (ok && e->conv2_tc) {
    const signed char *w2 = upload_padded_rows(e, m->conv2.w8, m->gru, 3 * m->cond, a.Kcp);   // natural [unit][K]
    ok = w2 && make_map_u8(&e->conv_maps.x, a.c2in, S, a.Kcp, TC_M) == 0 &&
         make_map_u8(&e->conv_maps.wi, w2, m->gru, a.Kcp, P_SLICE) == 0;
    e->conv_maps.h = e->conv_maps.x; e->conv_maps.wr = e->conv_maps.wi;
    ok = ok && cudaFuncSetAttribute(k_tc2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2_smem_bytes<false>(a.Kcp, m->gru)) == cudaSuccess;
  }
  // fused network kernel (net_kernel.cuh): needs the persistent wgmma GRU path and conv2 on the tensor cores
  // The fused kernel removes five launches and their drain/fill gaps per frame: it wins while the batch is latency-bound
  // and loses once the GPU is full, where its CTAs idle through the cluster barriers on SMs nothing else can share:
  // default up to 512 streams per device.
  // $RNNOISE_B200_NET_KERNEL = fused | layers overrides.
  {
    const char *nk = getenv("RNNOISE_B200_NET_KERNEL");
    const bool want = nk ? !strcmp(nk, "fused") : device_streams <= 512;
    e->net_fused = want && e->use_tc == 2 && e->conv2_tc;
  }
  {
    // CTAs per cluster of k_net.  8 halves every CTA's share of a layer (and the kernel's latency) but takes twice
    // the SMs per 128-stream tile: default 8 up to 8 tiles (1024 streams) on the device.  $RNNOISE_B200_NET_CLUSTER = 4 | 8 overrides.
    const char *nc = getenv("RNNOISE_B200_NET_CLUSTER");
    const int tiles = (device_streams + TC_M - 1) / TC_M;
    int want = nc ? atoi(nc) : tiles <= 8 ? 8 : 4;
    e->net_cluster = want == 8 && m->gru % (8 * P_SLICE) == 0 ? 8 : 4;
  }
  { const char *c1 = getenv("RNNOISE_B200_NET_CONV1"); e->net_conv1 = e->net_fused && !(c1 && !strcmp(c1, "0")); }
  if (ok && e->net_fused) {
    const size_t hs = Ss * m->gru, hs8 = Ss * a.Kp;
    for (int par = 0; par < 2; par++) {
      NetMaps &nm = e->net_maps[par];
      NetPtrs &np = e->net_ptrs[par];
      memset(&np, 0, sizeof(np));
      nm.x[0] = e->conv_maps.x; nm.wi[0] = e->conv_maps.wi; nm.h[0] = e->conv_maps.x; nm.wr[0] = e->conv_maps.wi;
      np.scale_i[0] = dm.conv2.scale; np.subias_i[0] = dm.conv2.subias;
      np.out_f32[0] = a.conv2_out + (size_t)par * hs; np.out_u8[0] = a.conv2_out_u8;
      if (e->net_conv1) {
        np.conv1_w = dm.conv1.w; np.conv1_b = dm.conv1.bias;
        np.features = a.features + (size_t)par * Ss * NB_FEATURES;
        np.conv1_state = a.conv1_state; np.c2in = a.c2in; np.cond = m->cond;
      }
      for (int l = 0; l < 3; l++) {
        const GruTcMaps &mp = e->tc_maps[par][l];
        nm.x[l + 1] = mp.x; nm.h[l + 1] = mp.h; nm.wi[l + 1] = mp.wi; nm.wr[l + 1] = mp.wr;
        np.scale_i[l + 1] = dm.gru_in[l].scale; np.subias_i[l + 1] = dm.gru_in[l].subias;
        np.scale_r[l + 1] = dm.gru_rec[l].scale; np.subias_r[l + 1] = dm.gru_rec[l].subias; np.diag[l + 1] = dm.gru_rec[l].diag;
        np.packed[l + 1] = dm.gru_rec[l].packed;
        np.h_old[l + 1] = a.hbuf + ((size_t)(par ^ 1) * 3 + l) * hs;
        np.out_f32[l + 1] = a.hbuf + ((size_t)par * 3 + l) * hs;
        np.out_u8[l + 1] = a.hbuf_u8 + ((size_t)par * 3 + l) * hs8;
      }
    }
    ok = cudaFuncSetAttribute(k_net, cudaFuncAttributeMaxDynamicSharedMemorySize, net_smem_bytes(a.Kcp, a.Kp, m->gru)) == cudaSuccess;
    if (!ok) fprintf(stderr, "[rnnoise_b200] fused network kernel setup failed\n");
  }
  if (!ok || cudaDeviceSynchronize() != cudaSuccess) {
    fprintf(stderr, "[rnnoise_b200] engine allocation/upload failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    b200_engine_destroy(e);
    return nullptr;
  }
  return e;
}

// Launch with (or without) the programmatic-dependent-launch attribute (see rnn_kernels.cuh).
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

extern "C" int b200_engine_streams(const B200Engine *e) { return e ? e->a.S : 0; }
extern "C" int b200_engine_ranges(const B200Engine *e) { return e ? e->nr : 0; }
// kernel launches of one frame: the five DSP kernels once per range, the network once for the whole batch
extern "C" int b200_engine_launches_per_frame(const B200Engine *e) {
  return !e ? NKERNELS : 5 * e->nr + (e->net_fused ? (e->net_conv1 ? 1 : 2) : 5);
}

// Parent-stream bracketing of device-pointer calls (lanes).  Only the kernels that touch the caller's
// buffers are ordered after the caller's stream -- the prefilter that reads the input, and the output heads /
// synthesis that write vad and PCM -- so the analysis and the network of the next frame never wait for the
// other lanes; the caller's stream waits for the call's completion (parent_leave).
static int parent_enter(B200Engine *e) {
  if (!e->parent) return 0;
  CK(cudaEventRecord(e->ev_pin, e->parent));
  return 0;
}
static bool tail_separate(const B200Engine *e) { return e->tail_overlap && e->overlap && !e->profiling; }
static cudaStream_t tail_stream(const B200Engine *e, int r) { return tail_separate(e) ? e->rg[r].s_tail : e->stream; }
// the caller's stream waits for the tails of the last frame handed to the engine
static int parent_leave(B200Engine *e) {
  if (!e->parent || e->frames < 1) return 0;
  const int par = (int)((e->frames - 1) & 1);
  for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(e->parent, e->rg[r].ev_back[par], 0));
  return 0;
}
static void launch_pitch(B200Engine *e, cudaStream_t st, int fr, int r0, int r1) {
  const int n = r1 - r0;
  if (e->pitch2)
    k_pitch2<<<(n + PG - 1) / PG, PG_THREADS, PITCH2_SMEM_BYTES, st>>>(e->a, fr, r0, r1);
  else
    k_pitch<<<(n + PITCH_NS - 1) / PITCH_NS, PITCH_NS * PITCH_THREADS, PITCH_NS * SM_PITCH_TOTAL * sizeof(float), st>>>(e->a, e->d_tables, fr, r0, r1);
}
static int frame_device_io(B200Engine *e, void *d_out, const void *d_in, float *d_vad, int s16);
extern "C" int b200_engine_frame_device(B200Engine *e, float *d_out, const float *d_in, float *d_vad) {
  if (!e || parent_enter(e) || frame_device_io(e, d_out, d_in, d_vad, 0)) return -1;
  return parent_leave(e);
}
extern "C" int b200_engine_frame_device_s16(B200Engine *e, short *d_out, const short *d_in, float *d_vad) {
  if (!e || parent_enter(e) || frame_device_io(e, d_out, d_in, d_vad, 1)) return -1;
  return parent_leave(e);
}
static int frame_device_io(B200Engine *e, void *d_out, const void *d_in, float *d_vad, int s16) {
  if (!e || !d_out || !d_in) return -1;
  CK(cudaSetDevice(e->device));
  const Arena &a = e->a;
  const int S = a.S, gru = a.gru, cond = a.cond;
  cudaStream_t st = e->stream;
  const int par = (int)(e->frames & 1);
  const size_t hstride = (size_t)S * gru, hstride8 = (size_t)S * a.Kp;
  float *h_new[3], *h_old[3];
  for (int l = 0; l < 3; l++) {
    h_new[l] = a.hbuf + ((size_t)par * 3 + l) * hstride;
    h_old[l] = a.hbuf + ((size_t)(par ^ 1) * 3 + l) * hstride;
  }
  // Three-stage software pipeline over streams: the analysis fronts (biquad -> k_pitch -> k_spectrum, one per range) of
  // frame f+1, the network of frame f on `st` (whole batch) and the tails (output heads -> synthesis, one per range) of
  // frame f-1 run side by side; each stage only waits for what it really depends on.  Hazards: xb[par] (ev_ana); the
  // spectrum slot f%3, features/silence[par], the GRU states and conv2 output of parity par, all last read by the tails
  // of frame f-2 (ev_back[par], recorded on the tails' streams).
  const bool overlap = e->overlap && !e->profiling;
  const bool tsep = tail_separate(e);
  float *c2o = a.conv2_out + (size_t)par * hstride;
  int ki = 0;
#define MARK() do { if (e->profiling) cudaEventRecord(e->ev[ki++], st); } while (0)
#define FRONT(R) (overlap ? (R).s_front : st)
  const int fr = frame_arg(e->frames);
  const int *sil = a.silence + (size_t)par * S;
  const float *feat = a.features + (size_t)par * S * NB_FEATURES;
  NvtxStages nv;
  nv.next("rnnoise_b200 frame: front (biquad, pitch, spectrum)");
  MARK();
  if (e->bq_frames > e->frames) {
    // the prefilter of this frame was issued ahead on the biquad streams (prefilter hint / pipelined
    // host call): just order the rest of the frame after it
    for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(FRONT(e->rg[r]), e->rg[r].ev_bq[par], 0));
  } else {
    // an engine driven directly on a caller's stream: the input is ordered on that stream (with the engine's own
    // stream the caller's work is ordered through the parent bracket, ev_pin, or not at all)
    const bool in_on_st = overlap && st != e->own_stream;
    if (in_on_st) CK(cudaEventRecord(e->ev_in, st));
    for (int r = 0; r < e->nr; r++) {
      B200Engine::Range &R = e->rg[r];
      cudaStream_t sf = FRONT(R);
      if (in_on_st) CK(cudaStreamWaitEvent(sf, e->ev_in, 0));
      if (overlap) CK(cudaStreamWaitEvent(sf, R.ev_bq[par ^ 1], 0));   // biquad state: after frame f-1's filter
      if (e->parent) CK(cudaStreamWaitEvent(sf, e->ev_pin, 0));
      k_biquad<<<(R.r1 - R.r0 + 31) / 32, 32, 0, sf>>>(a, d_in, fr, s16, e->io_stride, R.r0, R.r1);
      CK(cudaEventRecord(R.ev_bq[par], sf));
    }
    TL(e, e->frames, TL_BQ_END, FRONT(e->rg[0]));
    e->bq_frames = e->frames + 1;
  }
  MARK();
  for (int r = 0; r < e->nr; r++) {
    B200Engine::Range &R = e->rg[r];
    launch_pitch(e, FRONT(R), fr, R.r0, R.r1);
    CK(cudaEventRecord(R.ev_ana[par], FRONT(R)));   // xb[par] is free again
  }
  TL(e, e->frames, TL_PITCH_END, FRONT(e->rg[0]));
  MARK();
  for (int r = 0; r < e->nr; r++) {
    B200Engine::Range &R = e->rg[r];
    cudaStream_t sf = FRONT(R);
    if (overlap) CK(cudaStreamWaitEvent(sf, R.ev_back[par], 0));   // frame f-2 is done with slot f%3 / parity buffers
    k_spectrum<<<R.r1 - R.r0, DSP_THREADS, SM_SPEC_TOTAL * sizeof(float), sf>>>(a, e->d_tables, fr, R.r0);
    if (overlap) {
      CK(cudaEventRecord(R.ev_front[par], sf));
      CK(cudaStreamWaitEvent(st, R.ev_front[par], 0));
    }
  }
  TL(e, e->frames, TL_FRONT_END, FRONT(e->rg[0]));
  TL(e, e->frames, TL_BACK_START, st);
  nv.next("rnnoise_b200 frame: network (conv1, conv2, GRU x3)");
  MARK();
  const int gts = (S + RNN_TS - 1) / RNN_TS;
  if (tsep)   // the tails of frame f-2 have read the states of this parity
    for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(st, e->rg[r].ev_back[par], 0));
  if (!e->net_conv1) k_conv1<<<gts, 128, 0, st>>>(S, e->dm, feat, a.conv1_state, sil, a.c2in, a.Kcp);
  MARK();
  const bool pdl = e->pdl && !e->profiling;
  if (e->net_fused) {
    {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3((S + TC_M - 1) / TC_M, e->net_cluster); cfg.blockDim = dim3(P_THREADS);
      cfg.dynamicSmemBytes = net_smem_bytes(a.Kcp, a.Kp, gru); cfg.stream = st;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = e->net_cluster; attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      CK(cudaLaunchKernelEx(&cfg, k_net, S, a.Kcp, a.Kp, gru, e->net_maps[par], e->net_ptrs[par], sil));
    }
    MARK(); MARK(); MARK(); MARK();   // one launch covers the conv2 and GRU slots of the per-kernel profile
  } else {
    if (e->conv2_tc)
      CK(launch_pdl(k_tc2<false>, dim3((S + TC_M - 1) / TC_M, 4), dim3(P_THREADS), tc2_smem_bytes<false>(a.Kcp, gru), st, pdl,
                    S, a.Kcp, gru, a.Kp, e->conv_maps, e->dm.conv2, e->dm.conv2, (const float *)nullptr, c2o, a.conv2_out_u8, sil));
    else
      k_conv2<<<gts, 128, RNN_TS * (3 * cond / 4) * sizeof(uint32_t), st>>>(S, e->dm, a.c2in, a.Kcp, c2o, a.conv2_out_u8, a.Kp);
    MARK();
    const size_t gsm = 2 * RNN_TS * (gru / 4) * sizeof(uint32_t);
    for (int l = 0; l < 3; l++) {
      uint8_t *hu8_new = a.hbuf_u8 + ((size_t)par * 3 + l) * hstride8;
      if (e->use_tc == 2) {
        CK(launch_pdl(k_tc2<true>, dim3((S + TC_M - 1) / TC_M, 4), dim3(P_THREADS), tc2_smem_bytes<true>(a.Kp, gru), st, pdl,
                      S, a.Kp, gru, a.Kp, e->tc_maps[par][l], e->dm.gru_in[l], e->dm.gru_rec[l], (const float *)h_old[l], h_new[l], hu8_new, sil));
      } else if (e->use_tc == 1) {
        k_gru_tc<<<dim3((S + TC_M - 1) / TC_M, gru / TC_UNITS), 160, gru_tc_smem_bytes(gru), st>>>(
            S, gru, e->tc_maps[par][l], e->dm.gru_in[l], e->dm.gru_rec[l], h_old[l], h_new[l], hu8_new, sil);
      } else {
        const float *x = l == 0 ? c2o : h_new[l - 1];
        k_gru<<<dim3(gts, (gru + 127) / 128), 128, gsm, st>>>(S, gru, e->dm.gru_in[l], e->dm.gru_rec[l], x, h_old[l], h_new[l], hu8_new, a.Kp, sil);
      }
      MARK();
    }
  }
  if (tsep) CK(cudaEventRecord(e->ev_net[par], st));
  nv.next("rnnoise_b200 frame: tail (heads, synthesis)");
  const bool pdl_heads = pdl && e->use_tc == 2 && !e->net_fused && !tsep && e->nr == 1;   // only the k_tc2 predecessors are PDL-aware
  for (int r = 0; r < e->nr; r++) {
    B200Engine::Range &R = e->rg[r];
    cudaStream_t stl = tail_stream(e, r);
    const int n = R.r1 - R.r0;
    if (tsep) CK(cudaStreamWaitEvent(stl, e->ev_net[par], 0));
    if (e->parent) CK(cudaStreamWaitEvent(stl, e->ev_pin, 0));   // first kernel that writes the caller's buffers
    const float *c2 = c2o + (size_t)R.r0 * gru, *g1 = h_new[0] + (size_t)R.r0 * gru, *g2 = h_new[1] + (size_t)R.r0 * gru,
                *g3 = h_new[2] + (size_t)R.r0 * gru;
    float *gains = a.gains + (size_t)R.r0 * NB_BANDS, *vad = a.vad + R.r0;
    float *uvad = d_vad ? d_vad + (size_t)R.r0 * e->vad_stride : nullptr;
    const int *silr = sil + R.r0;
    if (e->heads2 && e->heads_ns == 1)
      CK(launch_pdl(k_heads2<1, 4>, dim3((n + 7) / 8), dim3(160), h2_smem_bytes<1>(), stl, pdl_heads, n, e->dm, c2, g1, g2, g3, silr, gains, vad, uvad, e->vad_stride));
    else if (e->heads2 && e->heads_ns == 2)
      CK(launch_pdl(k_heads2<2, 4>, dim3((n + 15) / 16), dim3(160), h2_smem_bytes<2>(), stl, pdl_heads, n, e->dm, c2, g1, g2, g3, silr, gains, vad, uvad, e->vad_stride));
    else if (e->heads2 && e->heads_ns == 8)
      CK(launch_pdl(k_heads2<2, 8>, dim3((n + 31) / 32), dim3(288), h2_smem_bytes<2, 8>(), stl, pdl_heads, n, e->dm, c2, g1, g2, g3, silr, gains, vad, uvad, e->vad_stride));
    else if (e->heads2)
      CK(launch_pdl(k_heads2<4, 4>, dim3((n + 31) / 32), dim3(160), h2_smem_bytes<4>(), stl, pdl_heads, n, e->dm, c2, g1, g2, g3, silr, gains, vad, uvad, e->vad_stride));
    else
      CK(launch_pdl(k_heads, dim3((n + HEAD_TS - 1) / HEAD_TS), dim3(160), 0, stl, pdl_heads, n, e->dm, c2, g1, g2, g3, silr, gains, vad, uvad, e->vad_stride));
  }
  MARK();
  for (int r = 0; r < e->nr; r++) {
    B200Engine::Range &R = e->rg[r];
    cudaStream_t stl = tail_stream(e, r);
    CK(launch_pdl(k_synthesis, dim3(R.r1 - R.r0), dim3(DSP_THREADS), SS_TOTAL * sizeof(float), stl, pdl_heads, a, (const DspTables *)e->d_tables, d_out, fr,
                  s16, e->io_stride, R.r0));
    CK(cudaEventRecord(R.ev_back[par], stl));
    // an engine driven directly on a caller's stream (no parent bracket): that stream sees the call complete
    if (stl != st && st != e->own_stream) CK(cudaStreamWaitEvent(st, R.ev_back[par], 0));
  }
  TL(e, e->frames, TL_BACK_END, tail_stream(e, 0));
  MARK();
#undef MARK
#undef FRONT
  CK(cudaGetLastError());
  e->frames++;
  if (e->profiling) {
    CK(cudaStreamSynchronize(st));
    for (int i = 0; i < NKERNELS; i++) {
      float ms = 0.f;
      CK(cudaEventElapsedTime(&ms, e->ev[i], e->ev[i + 1]));
      e->prof_ms[i] += ms;
    }
    e->prof_frames++;
  }
  return 0;
}

// Issue the high-pass prefilter of the next not-yet-prefiltered frame on the biquad streams.
// `ready` (optional) = event after which d_in is valid.  At most two frames ahead of processing.
static int issue_prefilter(B200Engine *e, const void *d_in, cudaEvent_t ready, int s16) {
  if (e->bq_frames >= e->frames + 2) return -1;
  const long long f = e->bq_frames;
  const int slot = (int)(f & 1);
  for (int r = 0; r < e->nr; r++) {
    B200Engine::Range &R = e->rg[r];
    if (ready) CK(cudaStreamWaitEvent(R.s_bq, ready, 0));
    CK(cudaStreamWaitEvent(R.s_bq, R.ev_ana[slot], 0));       // frame f-2 no longer reads this xb half
    CK(cudaStreamWaitEvent(R.s_bq, R.ev_bq[slot ^ 1], 0));    // biquad state: after frame f-1's filter
    k_biquad<<<(R.r1 - R.r0 + 31) / 32, 32, 0, R.s_bq>>>(e->a, d_in, frame_arg(f), s16, e->io_stride, R.r0, R.r1);
    CK(cudaGetLastError());
    CK(cudaEventRecord(R.ev_bq[slot], R.s_bq));
  }
  TL(e, f, TL_BQ_END, e->rg[0].s_bq);
  e->bq_frames = f + 1;
  return 0;
}

extern "C" int b200_engine_prefilter_ahead(const B200Engine *e) { return e ? (int)(e->bq_frames - e->frames) : 0; }
extern "C" int b200_engine_prefilter_device(B200Engine *e, const float *d_in) {
  if (!e || !d_in) return -1;
  CK(cudaSetDevice(e->device));
  return issue_prefilter(e, d_in, nullptr, 0);
}

static int frame_host_async_io(B200Engine *e, void *out, const void *in, float *vad, int s16) {
  if (!e || !out || !in) return -1;
  if (e->bq_frames != e->frames) return -1;   // a device-side prefilter hint is pending: do not mix
  NVTX_SCOPE("rnnoise_b200 host frame (H2D, frame, D2H enqueue)");
  CK(cudaSetDevice(e->device));
  const size_t n = (size_t)e->a.S * FRAME_SIZE * (s16 ? sizeof(short) : sizeof(float));
  const int slot = (int)(e->host_frames & 1), par = (int)(e->frames & 1);
  // copy-in: the staging slot is free once the prefilters of frame n-2 have consumed it
  for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(e->s_h2d, e->rg[r].ev_bq[par], 0));
  TL(e, e->frames, TL_H2D_START, e->s_h2d);
  CK(cudaMemcpyAsync(e->stage_in[slot], in, n, cudaMemcpyHostToDevice, e->s_h2d));
  CK(cudaEventRecord(e->ev_h2d[slot], e->s_h2d));
  TL(e, e->frames, TL_H2D_END, e->s_h2d);
  // high-pass prefilter on its own stream: overlaps the previous frame's kernels
  if (issue_prefilter(e, e->stage_in[slot], e->ev_h2d[slot], s16)) return -1;
  // rest of the frame: needs frame n-2's output staging drained
  for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(tail_stream(e, r), e->ev_d2h[slot], 0));   // the tails write the output staging
  if (frame_device_io(e, e->stage_out[slot], e->stage_in[slot], e->stage_vad[slot], s16)) return -1;
  // copy-out: after the tails of every range
  for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(e->s_d2h, e->rg[r].ev_back[par], 0));
  CK(cudaMemcpyAsync(out, e->stage_out[slot], n, cudaMemcpyDeviceToHost, e->s_d2h));
  if (vad) CK(cudaMemcpyAsync(vad, e->stage_vad[slot], (size_t)e->a.S * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
  CK(cudaEventRecord(e->ev_d2h[slot], e->s_d2h));
  TL(e, e->frames - 1, TL_D2H_END, e->s_d2h);
  e->host_frames++;
  return 0;
}
extern "C" int b200_engine_frame_host_async(B200Engine *e, float *out, const float *in, float *vad) {
  return frame_host_async_io(e, out, in, vad, 0);
}
extern "C" int b200_engine_frame_host_async_s16(B200Engine *e, short *out, const short *in, float *vad) {
  return frame_host_async_io(e, out, in, vad, 1);
}

// ------------------------------------------------------------------------------------------------
// Multi-frame calls (SURVEY 8(f) rank 2): T consecutive frames of every stream per call.  Buffers hold
// each stream's audio contiguously, pcm[s][t * 480 + i] and vad[s][t] -- the layout of a decoded file --
// so the kernels index streams with a stride of T * 480 (T for vad).  Results are bit-identical to T
// frame-at-a-time calls: the same kernels run in the same order on the same state.
// ------------------------------------------------------------------------------------------------
static int frames_device_io(B200Engine *e, void *d_out, const void *d_in, float *d_vad, int T, int pcm_stride,
                            int vad_stride, int s16) {
  if (!e || !d_out || !d_in || T < 1 || e->bq_frames != e->frames) return -1;
  const size_t esz = s16 ? sizeof(short) : sizeof(float);
  const char *in = (const char *)d_in;
  char *out = (char *)d_out;
  NVTX_SCOPE("rnnoise_b200 multi-frame call");
  e->io_stride = pcm_stride;
  e->vad_stride = vad_stride;
  int rc = 0;
  // the high-pass prefilter runs up to two frames ahead on its own stream (the input is all there);
  // it is ordered after the caller's stream once, through ev_in
  // (the engine's own stream may itself be waiting for a staging copy of the host path: always order after it;
  //  with a parent stream, additionally after the caller's stream)
  rc = cudaEventRecord(e->ev_in, e->stream) != cudaSuccess;
  for (int r = 0; r < e->nr && !rc && e->parent; r++) rc = cudaStreamWaitEvent(e->rg[r].s_bq, e->ev_pin, 0) != cudaSuccess;
  for (int t = 0; t < 2 && t < T && !rc; t++) rc = issue_prefilter(e, in + (size_t)t * FRAME_SIZE * esz, t == 0 ? e->ev_in : nullptr, s16);
  for (int t = 0; t < T && !rc; t++) {
    rc = frame_device_io(e, out + (size_t)t * FRAME_SIZE * esz, in + (size_t)t * FRAME_SIZE * esz, d_vad ? d_vad + t : nullptr, s16);
    if (!rc && t + 2 < T) rc = issue_prefilter(e, in + (size_t)(t + 2) * FRAME_SIZE * esz, nullptr, s16);
  }
  e->io_stride = FRAME_SIZE;
  e->vad_stride = 1;
  return rc ? -1 : 0;
}
extern "C" int b200_engine_frames_device(B200Engine *e, void *d_out, const void *d_in, float *d_vad, int T, int s16) {
  if (!e) return -1;
  CK(cudaSetDevice(e->device));
  if (parent_enter(e) || frames_device_io(e, d_out, d_in, d_vad, T, T * FRAME_SIZE, T, s16)) return -1;
  return parent_leave(e);
}

// Host buffers: the T frames move in chunks of `multi_chunk` frames through double-buffered device
// staging ([S][chunk * 480]), strided 2-D copies on the copy streams, so H2D(c+1), kernels(c) and
// D2H(c-1) overlap.  Blocking: returns when `out` and `vad` are complete.
extern "C" int b200_engine_frames_host_enqueue(B200Engine *e, void *out, const void *in, float *vad, int T, int s16, int pitch_frames) {
  if (!e || !out || !in || T < 1 || e->bq_frames != e->frames) return -1;
  CK(cudaSetDevice(e->device));
  const size_t S = (size_t)e->a.S, esz = s16 ? sizeof(short) : sizeof(float);
  const int C = T < e->multi_chunk ? T : e->multi_chunk;
  const size_t need = S * C * FRAME_SIZE * sizeof(float);   // sized for float so both sample types fit
  if (need > e->multi_bytes) {
    CK(cudaDeviceSynchronize());
    for (int i = 0; i < 2; i++) {
      cudaFree(e->multi_in[i]); cudaFree(e->multi_out[i]); cudaFree(e->multi_vad[i]);
      e->multi_in[i] = e->multi_out[i] = nullptr; e->multi_vad[i] = nullptr;
    }
    e->multi_bytes = 0;
    for (int i = 0; i < 2; i++) {
      CK(cudaMalloc(&e->multi_in[i], need));
      CK(cudaMalloc(&e->multi_out[i], need));
      CK(cudaMalloc(&e->multi_vad[i], S * C * sizeof(float)));
    }
    e->multi_bytes = need;
  }
  const size_t host_pitch = (size_t)pitch_frames * FRAME_SIZE * esz;   // = T for a whole buffer
  int c = 0;
  for (int t0 = 0; t0 < T; t0 += C, c++) {
    const int n = T - t0 < C ? T - t0 : C, slot = c & 1;
    const size_t dev_pitch = (size_t)n * FRAME_SIZE * esz;
    // copy-in once chunk c-2's kernels have read this slot
    CK(cudaStreamWaitEvent(e->s_h2d, e->ev_mcomp[slot], 0));
    CK(cudaMemcpy2DAsync(e->multi_in[slot], dev_pitch, (const char *)in + (size_t)t0 * FRAME_SIZE * esz, host_pitch,
                         dev_pitch, S, cudaMemcpyHostToDevice, e->s_h2d));
    CK(cudaEventRecord(e->ev_mh2d[slot], e->s_h2d));
    // kernels: after the copy-in, and after chunk c-2's copy-out has drained the output slot
    CK(cudaStreamWaitEvent(e->stream, e->ev_mh2d[slot], 0));
    for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(tail_stream(e, r), e->ev_md2h[slot], 0));
    if (frames_device_io(e, e->multi_out[slot], e->multi_in[slot], e->multi_vad[slot], n, n * FRAME_SIZE, n, s16)) return -1;
    // copy-out: after the tails of the chunk's last frame (which follow everything else of the chunk)
    for (int r = 0; r < e->nr; r++) CK(cudaStreamWaitEvent(e->s_d2h, e->rg[r].ev_back[(e->frames - 1) & 1], 0));
    CK(cudaEventRecord(e->ev_mcomp[slot], e->s_d2h));
    CK(cudaMemcpy2DAsync((char *)out + (size_t)t0 * FRAME_SIZE * esz, host_pitch, e->multi_out[slot], dev_pitch,
                         dev_pitch, S, cudaMemcpyDeviceToHost, e->s_d2h));
    if (vad)
      CK(cudaMemcpy2DAsync(vad + t0, (size_t)pitch_frames * sizeof(float), e->multi_vad[slot], (size_t)n * sizeof(float),
                           (size_t)n * sizeof(float), S, cudaMemcpyDeviceToHost, e->s_d2h));
    CK(cudaEventRecord(e->ev_md2h[slot], e->s_d2h));
  }
  return 0;
}
extern "C" int b200_engine_frames_host(B200Engine *e, void *out, const void *in, float *vad, int T, int s16) {
  if (b200_engine_frames_host_enqueue(e, out, in, vad, T, s16, T)) return -1;
  return b200_engine_sync(e);
}

// ------------------------------------------------------------------------------------------------
// Training-feature extraction (SURVEY 8(f) rank 4): the frame loop of src/dump_features.c:466-491 for
// every stream of the batch.  The noisy frame goes through the pitch + spectrum kernels with the
// reference's TRAINING semantics (no high-pass prefilter: dump_features filters whole sequences itself,
// :421-432), the clean frame through a window + FFT + band-energy pass; out = [S][98] records.
// A batch used this way keeps its own signal history; do not interleave with denoising calls.
// ------------------------------------------------------------------------------------------------
extern "C" int b200_engine_train_features_device(B200Engine *e, float *d_rec, const float *d_clean, const float *d_noisy,
                                                 const float *d_vad_target, const int *d_noise_free, const int *d_lowpass,
                                                 const int *d_band_lp) {
  if (!e || !d_rec || !d_clean || !d_noisy || e->bq_frames != e->frames) return -1;
  CK(cudaSetDevice(e->device));
  if (parent_enter(e)) return -1;
  const Arena &a = e->a;
  const size_t S = (size_t)a.S;
  cudaStream_t st = e->stream;
  if (e->parent) CK(cudaStreamWaitEvent(st, e->ev_pin, 0));
  if (!e->train_clean_mem) {
    CK(cudaMalloc(&e->train_clean_mem, S * FRAME_SIZE * sizeof(float)));
    e->allocs.push_back(e->train_clean_mem);
    CK(cudaMemsetAsync(e->train_clean_mem, 0, S * FRAME_SIZE * sizeof(float), st));
  }
  // order after whatever the analysis streams of earlier denoising calls still run
  for (int r = 0; r < e->nr; r++)
    for (int i = 0; i < 2; i++) {
      CK(cudaStreamWaitEvent(st, e->rg[r].ev_ana[i], 0));
      CK(cudaStreamWaitEvent(st, e->rg[r].ev_front[i], 0));
      CK(cudaStreamWaitEvent(st, e->rg[r].ev_back[i], 0));
    }
  const int par = (int)(e->frames & 1), fr = frame_arg(e->frames);
  CK(cudaMemcpyAsync(a.xb + (size_t)par * S * FRAME_SIZE, d_noisy, S * FRAME_SIZE * sizeof(float), cudaMemcpyDeviceToDevice, st));
  launch_pitch(e, st, fr, 0, a.S);
  TrainIo io;
  io.clean = d_clean; io.clean_mem = e->train_clean_mem; io.rec = d_rec;
  io.vad_target = d_vad_target; io.noise_free = d_noise_free; io.lowpass = d_lowpass; io.band_lp = d_band_lp;
  k_train_features<<<a.S, DSP_THREADS, SM_SPEC_TOTAL * sizeof(float), st>>>(a, e->d_tables, fr, io);
  CK(cudaGetLastError());
  for (int r = 0; r < e->nr; r++) {   // later denoising-style calls order after this one through the usual events
    CK(cudaEventRecord(e->rg[r].ev_ana[par], st));
    CK(cudaEventRecord(e->rg[r].ev_front[par], st));
    CK(cudaEventRecord(e->rg[r].ev_back[par], st));
  }
  e->frames++;
  e->bq_frames = e->frames;
  e->host_frames = e->frames;
  return parent_leave(e);   // (waits for ev_back of this call's parity: recorded above on the engine's stream)
}

extern "C" int b200_engine_train_features_host(B200Engine *e, float *rec, const float *clean, const float *noisy,
                                               const float *vad_target, const int *noise_free, const int *lowpass, const int *band_lp) {
  if (!e || !rec || !clean || !noisy) return -1;
  CK(cudaSetDevice(e->device));
  const size_t S = (size_t)e->a.S, F = S * FRAME_SIZE;
  if (!e->train_stage) {
    CK(cudaMalloc(&e->train_stage, (2 * F + S * TRAIN_RECORD + 4 * S) * sizeof(float)));
    e->allocs.push_back(e->train_stage);
  }
  float *d_clean = e->train_stage, *d_noisy = d_clean + F, *d_rec = d_noisy + F, *d_vt = d_rec + S * TRAIN_RECORD;
  int *d_nf = (int *)(d_vt + S), *d_lp = d_nf + S, *d_bl = d_lp + S;
  cudaStream_t st = e->stream;
  CK(cudaMemcpyAsync(d_clean, clean, F * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_noisy, noisy, F * sizeof(float), cudaMemcpyHostToDevice, st));
  if (vad_target) CK(cudaMemcpyAsync(d_vt, vad_target, S * sizeof(float), cudaMemcpyHostToDevice, st));
  if (noise_free) CK(cudaMemcpyAsync(d_nf, noise_free, S * sizeof(int), cudaMemcpyHostToDevice, st));
  if (lowpass) CK(cudaMemcpyAsync(d_lp, lowpass, S * sizeof(int), cudaMemcpyHostToDevice, st));
  if (band_lp) CK(cudaMemcpyAsync(d_bl, band_lp, S * sizeof(int), cudaMemcpyHostToDevice, st));
  if (b200_engine_train_features_device(e, d_rec, d_clean, d_noisy, vad_target ? d_vt : nullptr, noise_free ? d_nf : nullptr,
                                        lowpass ? d_lp : nullptr, band_lp ? d_bl : nullptr)) return -1;
  CK(cudaMemcpyAsync(rec, d_rec, S * TRAIN_RECORD * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int b200_engine_frame_host(B200Engine *e, float *out, const float *in, float *vad) {
  if (b200_engine_frame_host_async(e, out, in, vad)) return -1;
  CK(cudaStreamSynchronize(e->s_d2h));
  return 0;
}

extern "C" int b200_engine_sync(B200Engine *e) {
  if (!e) return -1;
  NVTX_SCOPE("rnnoise_b200 sync");
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize(e->s_h2d));
  for (int r = 0; r < e->nr; r++) { CK(cudaStreamSynchronize(e->rg[r].s_bq)); CK(cudaStreamSynchronize(e->rg[r].s_front)); }
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));
  CK(cudaStreamSynchronize(e->s_d2h));
  return 0;
}

extern "C" int b200_engine_set_stream(B200Engine *e, void *cuda_stream) {
  if (!e) return -1;
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));
  e->stream = cuda_stream ? (cudaStream_t)cuda_stream : e->own_stream;
  return 0;
}

// Lane mode: keep the engine's own stream, but bracket device-pointer calls with `parent` (NULL: off).
extern "C" int b200_engine_set_parent(B200Engine *e, void *parent_stream) {
  if (!e) return -1;
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));
  e->stream = e->own_stream;
  e->parent = (cudaStream_t)parent_stream;
  return 0;
}

extern "C" int b200_engine_profile(B200Engine *e, int enable) {
  if (!e) return -1;
  CK(cudaSetDevice(e->device));
  if (b200_engine_sync(e)) return -1;   // the stream roles change with the profiling flag: drain every stage first
  if (enable) {
    for (int i = 0; i <= NKERNELS; i++) if (!e->ev[i]) CK(cudaEventCreate(&e->ev[i]));
    for (int i = 0; i < NKERNELS; i++) e->prof_ms[i] = 0.0;
    e->prof_frames = 0;
  }
  e->profiling = enable ? 1 : 0;
  return 0;
}

extern "C" int b200_engine_profile_read(B200Engine *e, float *ms, const char **names, int capacity, int *frames) {
  if (!e || !ms || capacity < NKERNELS) return -1;
  for (int i = 0; i < NKERNELS; i++) {
    ms[i] = (float)e->prof_ms[i];
    if (names) names[i] = e->net_fused && i == 4 ? "k_net" : (e->net_fused && i >= 5 && i <= 7) || (e->net_conv1 && i == 3) ? "-" : kKernelNames[i];
  }
  if (frames) *frames = e->prof_frames;
  return NKERNELS;
}

// [frames recorded][TL_POINTS] milliseconds since the first recorded point; NaN where a point was not recorded
extern "C" int b200_engine_timeline_read(B200Engine *e, float *dst, int capacity) {
  if (!e || !dst) return -1;
  if (b200_engine_sync(e)) return -1;
  const int nf = (int)(e->frames < e->tl_frames ? e->frames : e->tl_frames);
  if (capacity < nf * TL_POINTS) return -1;
  cudaEvent_t t0 = nullptr;
  for (int i = 0; i < TL_POINTS && !t0 && nf > 0; i++)
    if (cudaEventQuery(e->tl[i]) == cudaSuccess) { float x; if (cudaEventElapsedTime(&x, e->tl[i], e->tl[i]) == cudaSuccess) t0 = e->tl[i]; }
  cudaGetLastError();
  for (int i = 0; i < nf * TL_POINTS; i++) {
    float ms = 0.f;
    dst[i] = t0 && cudaEventElapsedTime(&ms, t0, e->tl[i]) == cudaSuccess ? ms : nanf("");
  }
  cudaGetLastError();
  return nf;
}

extern "C" int b200_engine_reset_stream(B200Engine *e, int s) {
  if (!e || s < 0 || s >= e->a.S) return -1;
  if (e->bq_frames != e->frames) return -1;   // a prefilter hint already consumed the old filter state for the next frame
  CK(cudaSetDevice(e->device));
  const Arena &a = e->a;
  const size_t S = a.S;
  cudaStream_t st = e->stream;
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));   // the tails of the last frame still read / write this stream's state
#define ZERO(ptr, per, copies)                                                                          \
  for (int c_ = 0; c_ < (copies); c_++)                                                                 \
    CK(cudaMemsetAsync((ptr) + ((size_t)c_ * S + s) * (per), 0, (size_t)(per) * sizeof(*(ptr)), st));
  ZERO(a.ring, PITCH_BUF_SIZE, 1) ZERO(a.synth_mem, FRAME_SIZE, 1) ZERO(a.hp_mem, 2, 1)
  ZERO(a.spec, 4 * FREQ_SIZE, 3) ZERO(a.band, 96, 3) ZERO(a.lastg, NB_BANDS, 1) ZERO(a.pitch_state, 2, 1)
  ZERO(a.conv1_state, 2 * NB_FEATURES, 1) ZERO(a.hbuf, a.gru, 6)
#undef ZERO
  for (int c = 0; c < 6; c++) CK(cudaMemsetAsync(a.hbuf_u8 + ((size_t)c * S + s) * a.Kp, 127, a.Kp, st));
  CK(cudaMemsetAsync(a.c2in + (size_t)s * a.Kcp, 127, a.Kcp, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

#ifdef PITCH_TIMING
// diagnostics build only: clock64() stamps of one CTA of the last k_pitch2 launch (start, then after each phase)
extern "C" __attribute__((visibility("default"))) int b200_debug_pitch_timing(long long *dst, int n) {
  if (n > 32) n = 32;
  cudaDeviceSynchronize();
  return cudaMemcpyFromSymbol(dst, g_pitch_t, n * sizeof(long long)) == cudaSuccess ? n : -1;
}
#endif

// Test hook: start a FRESH engine (all state zero, nothing enqueued) at an arbitrary frame index, so the
// counter wrap can be crossed in a few frames.  Fails once a frame has been processed.
extern "C" int b200_engine_debug_set_frames(B200Engine *e, long long frames) {
  if (!e || frames < 0 || e->frames != 0 || e->bq_frames != 0 || e->host_frames != 0) return -1;
  e->frames = e->bq_frames = e->host_frames = frames;
  return 0;
}

// Bulk form for long parity statistics: item `what` of EVERY stream, [S][n] floats (pitch: {period, gain};
// silence: 0/1; features: 65).  Returns n or -1.
extern "C" int b200_engine_debug_read_all(B200Engine *e, int what, float *dst, int cap) {
  if (!e || !dst || e->frames < 1) return -1;
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));
  const Arena &a = e->a;
  const size_t S = a.S;
  const int par = frame_arg(e->frames - 1) & 1;
  const void *src; int n;
  switch (what) {
    case RNNOISE_DBG_PITCH: src = a.pitch_state; n = 2; break;
    case RNNOISE_DBG_SILENCE: src = a.silence + (size_t)par * S; n = 1; break;
    case RNNOISE_DBG_FEATURES: src = a.features + (size_t)par * S * NB_FEATURES; n = NB_FEATURES; break;
    case RNNOISE_DBG_GAINS: src = a.gains; n = NB_BANDS; break;
    default: return -1;
  }
  if ((size_t)cap < S * n) return -1;
  CK(cudaMemcpy(dst, src, S * n * sizeof(float), cudaMemcpyDeviceToHost));
  if (what == RNNOISE_DBG_PITCH) for (size_t s = 0; s < S; s++) { int p; memcpy(&p, dst + 2 * s, 4); dst[2 * s] = (float)p; }
  if (what == RNNOISE_DBG_SILENCE) for (size_t s = 0; s < S; s++) { int p; memcpy(&p, dst + s, 4); dst[s] = (float)p; }
  return n;
}

extern "C" int b200_engine_debug_read(B200Engine *e, int what, int s, float *dst, int cap) {
  if (!e || !dst || s < 0 || s >= e->a.S || e->frames < 1) return -1;
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < e->nr; r++) CK(cudaStreamSynchronize(e->rg[r].s_tail));
  const Arena &a = e->a;
  const size_t S = a.S;
  const int fl = frame_arg(e->frames - 1);   // the index the kernels of the last frame were handed
  const int par = fl & 1, slot = fl % 3;
  const float *src = nullptr;
  int n = 0;
  switch (what) {
    case RNNOISE_DBG_FEATURES: src = a.features + ((size_t)par * S + s) * NB_FEATURES; n = NB_FEATURES; break;
    case RNNOISE_DBG_X: src = a.spec + ((size_t)slot * S + s) * 4 * FREQ_SIZE; n = 2 * FREQ_SIZE; break;
    case RNNOISE_DBG_P: src = a.spec + ((size_t)slot * S + s) * 4 * FREQ_SIZE + 2 * FREQ_SIZE; n = 2 * FREQ_SIZE; break;
    case RNNOISE_DBG_EX: src = a.band + ((size_t)slot * S + s) * 96; n = 32; break;
    case RNNOISE_DBG_EP: src = a.band + ((size_t)slot * S + s) * 96 + 32; n = 32; break;
    case RNNOISE_DBG_EXP: src = a.band + ((size_t)slot * S + s) * 96 + 64; n = 32; break;
    case RNNOISE_DBG_GAINS: src = a.gains + (size_t)s * NB_BANDS; n = NB_BANDS; break;
    case RNNOISE_DBG_LASTG: src = a.lastg + (size_t)s * NB_BANDS; n = NB_BANDS; break;
    case RNNOISE_DBG_XB: src = a.xb + ((size_t)par * S + s) * FRAME_SIZE; n = FRAME_SIZE; break;
    case RNNOISE_DBG_GRU1: case RNNOISE_DBG_GRU2: case RNNOISE_DBG_GRU3:
      src = a.hbuf + (((size_t)par * 3 + (what - RNNOISE_DBG_GRU1)) * S + s) * a.gru; n = a.gru; break;
    case RNNOISE_DBG_CONV1_STATE: src = a.conv1_state + (size_t)s * 2 * NB_FEATURES; n = 2 * NB_FEATURES; break;
    case RNNOISE_DBG_CONV2_STATE: {   // kept as u8 (the only form conv2 consumes): returned as floats 0..255.
      // After a frame the operand row is [memory the frame saw (2 x cond) | the frame's conv1 output (cond)]; the
      // reference's conv2_state at that point (nnet.c:122: mem = tmp[in_size:]) is the LAST 2 x cond entries.
      n = 2 * a.cond;
      if (cap < n) return -1;
      std::vector<uint8_t> tmp(n);
      CK(cudaMemcpy(tmp.data(), a.c2in + (size_t)s * a.Kcp + a.cond, n, cudaMemcpyDeviceToHost));
      for (int i = 0; i < n; i++) dst[i] = (float)tmp[i];
      return n;
    }
    case RNNOISE_DBG_PITCH: src = a.pitch_state + 2 * (size_t)s; n = 2; break;
    case RNNOISE_DBG_SILENCE: src = (const float *)(a.silence + (size_t)par * S + s); n = 1; break;
    case RNNOISE_DBG_CONV2_OUT: src = a.conv2_out + ((size_t)par * S + s) * a.gru; n = a.gru; break;
    default: return -1;
  }
  if (cap < n) return -1;
  CK(cudaMemcpy(dst, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  if (what == RNNOISE_DBG_PITCH) { int p; memcpy(&p, dst, 4); dst[0] = (float)p; }
  if (what == RNNOISE_DBG_SILENCE) { int p; memcpy(&p, dst, 4); dst[0] = (float)p; }
  return n;
}
