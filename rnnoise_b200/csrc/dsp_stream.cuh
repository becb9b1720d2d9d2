// dsp_stream.cuh -- the two per-stream DSP bodies (analysis before the network, synthesis after).
// See dsp_core.cuh for the execution model (PHASE = barrier-separated step of a 128-thread CTA,
// or a loop over tid in the host emulation used by tests/emu).
#pragma once
#include "dsp_core.cuh"

#if defined(__CUDA_ARCH__)
#define PHASE_BEGIN { const int tid = threadIdx.x; const int nthr = DSP_THREADS; (void)nthr;
#define PHASE_END } __syncthreads();
#else
#define PHASE_BEGIN for (int tid = 0; tid < DSP_THREADS; ++tid) { const int nthr = DSP_THREADS; (void)nthr;
#define PHASE_END }
#endif

struct PitchArgs {
  const float *xb;      // [480]  this stream's frame after the high-pass biquad
  float *ring;          // [1728] pitch-history ring of this stream
  int ring_base;        // physical index of logical sample 0 AFTER this frame's 480-sample shift
  float *pitch_state;   // [2] {last_period as int bits, last_gain}: read as the prior, then updated
};
struct SpectrumArgs {
  const float *ring;    // [1728] ring, already holding this frame
  int ring_base;
  const float *pitch_state; // [2] this frame's pitch period (int bits) from the pitch kernel
  float *spec_out;      // [2][962] X then P of this frame (becomes "delayed" next frame)
  float *band_out;      // [3][32]  Ex, Ep, Exp
  float *features;      // [65]
  int *silence;         // [1]
  int lowpass;          // TRAIN only: bins >= lowpass of X are zeroed (denoise.c:340-343)
};

// Pitch half of rnn_compute_frame_features (src/denoise.c:359-370): rnn_pitch_downsample /
// rnn_pitch_search / rnn_remove_doubling (src/pitch.c:146,281,423) for PITCH_NS streams per CTA.
//
// The pitch analysis is dominated by SERIAL float chains (each lag's dot product, the running
// energies, the selection scans) that occupy 1..10 lanes of a warp.  A CTA therefore owns PITCH_NS
// streams: phases whose work is wide (decimation, FIR, the 30-lane correlations) run on the 128
// threads of each stream's own warp quartet, while the narrow chains of ALL the CTA's streams are
// packed side by side into the lanes of one or two warps -- same instructions, PITCH_NS x the useful
// lanes.  Thread ids: q = tid / PITCH_THREADS is the stream a thread belongs to, t its local id;
// packed phases use the first lanes of the CTA instead.
// 96 threads per stream and PITCH_NS 4: 5 CTAs x 4 = 20 streams resident per SM (the thread-slot limit; with one stream
// per CTA the 1 KB the hardware reserves per CTA costs two of them).  128 threads per stream leave 16 streams per SM.
#ifndef PITCH_NS
#define PITCH_NS 4
#endif
// Threads per stream in the pitch kernel.  The chains keep one warp busy per stream, so more resident
// streams per SM hide more latency: 96 threads (3 warps) x 20 streams fill an SM's 2048 thread slots
// and its shared memory (20 x 11.3 KB), against 16 streams with 128 threads.
#ifndef PITCH_THREADS
#define PITCH_THREADS 96
#endif
static_assert(PITCH_THREADS >= 96 && PITCH_THREADS % 32 == 0, "phases use local thread ids up to 64 + PITCH_NS");
#if defined(__CUDA_ARCH__)
#define MPHASE_BEGIN { const int tid = threadIdx.x; const int q = tid / PITCH_THREADS, t = tid % PITCH_THREADS; (void)q; (void)t;
#define MPHASE_END } __syncthreads();
#else
#define MPHASE_BEGIN for (int tid = 0; tid < PITCH_NS * PITCH_THREADS; ++tid) { const int q = tid / PITCH_THREADS, t = tid % PITCH_THREADS; (void)q; (void)t;
#define MPHASE_END }
#endif
#define PSM(qq) (sm + (qq) * SM_PITCH_TOTAL)
#ifndef PITCH_CHAIN4
#define PITCH_CHAIN4 1
#endif

// a[q].ring == nullptr marks an absent stream (batch size not a multiple of PITCH_NS)
HD void pitch_streams(float *sm, const PitchArgs *a, const DspTables *T) {
  (void)T;
  // -- the updated 1728-sample history [old ring part | this frame] (denoise.c:359-360; a ring instead of the memmove)
  //    is fetched ONCE, in logical order, into the space of the two half-rate signals (dead until the decimation has
  //    run): 432 aligned 16-byte asynchronous copies per stream, all of a thread's requests in flight together, L1
  //    bypassed -- one HBM / L2 round trip for the phase (the CTAs of an SM run it in lock-step, so nothing else hides
  //    the latency; the register version paid four dependent round trips and 32 load instructions per thread).
  MPHASE_BEGIN
    if (a[q].ring) {
      const PitchArgs A = a[q];
      float *raw = PSM(q) + SM_LP;
      const int H = PITCH_BUF_SIZE - FRAME_SIZE;
      static_assert(SM_LP == 0 && SM_LP0 == LP_SIZE && 2 * LP_SIZE == PITCH_BUF_SIZE && SM_PITCH_TOTAL % 4 == 0, "raw history over lp | lp0");
      static_assert((PITCH_BUF_SIZE - FRAME_SIZE) % 4 == 0, "a piece is either old history or new frame");
      for (int c = t; c < PITCH_BUF_SIZE / 4; c += PITCH_THREADS) {
        const int k = 4 * c;   // ring base and ring length are multiples of 4 floats: a piece never straddles the ring's end
        async_copy16(raw + k, k < H ? A.ring + ring_pos(A.ring_base, k) : A.xb + (k - H));
      }
    }
    async_wait_all();
  MPHASE_END
  // -- append the new frame to the ring (the 480 slots being overwritten hold the oldest samples, which nothing reads
  //    any more) and decimate by 2 (pitch.c:171-173) into the scratch that the searches use later
  MPHASE_BEGIN
    if (a[q].ring) {
      const PitchArgs A = a[q];
      const float *raw = PSM(q) + SM_LP;
      float *lp0 = PSM(q) + SM_LP0N;
      const int H = PITCH_BUF_SIZE - FRAME_SIZE;
      for (int j = t; j < FRAME_SIZE; j += PITCH_THREADS) {
        int p = A.ring_base + H + j; if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
        A.ring[p] = raw[H + j];
      }
      for (int i = t; i < LP_SIZE; i += PITCH_THREADS) {
        const float c = raw[2 * i], r = raw[2 * i + 1];
        lp0[i] = i ? .5f * (.5f * (raw[2 * i - 1] + r) + c) : .5f * (.5f * r + c);
      }
    }
  MPHASE_END
  // -- autocorrelation lags 0..4 (celt_lpc.c:92-174: first n-4 samples, then the tail): 5 lanes per
  //    stream, all streams packed into warp 0 (lane = 8 * stream + lag)
  MPHASE_BEGIN
    if (tid < 8 * PITCH_NS && (tid & 7) < 5 && a[tid >> 3].ring) {
      const int qq = tid >> 3, k = tid & 7, fastN = LP_SIZE - 4;
      const float *lp0 = PSM(qq) + SM_LP0N;
#if PITCH_CHAIN4
      const float s = dot_chain4(0.f, lp0, lp0 + k, fastN);
#else
      float s = 0.f;
#pragma unroll 4
      for (int j = 0; j < fastN; j++) s = s + lp0[j] * lp0[j + k];
#endif
      float d = 0.f;
      for (int i = k + fastN; i < LP_SIZE; i++) d = d + lp0[i] * lp0[i - k];
      PSM(qq)[SM_PITCH_END + MI_AC + k] = s + d;
    }
  MPHASE_END
  MPHASE_BEGIN
    if (tid < PITCH_NS && a[tid].ring) lpc_taps(PSM(tid) + SM_PITCH_END + MI_AC, PSM(tid) + SM_PITCH_END + MI_NUM);
  MPHASE_END
  // -- 5-tap whitening FIR with zero history (celt_fir5, pitch.c:104-143)
  MPHASE_BEGIN
    if (a[q].ring) {
      const float *lp0 = PSM(q) + SM_LP0N, *num = PSM(q) + SM_PITCH_END + MI_NUM;
      float *lp = PSM(q) + SM_LP;
      for (int i = t; i < LP_SIZE; i += PITCH_THREADS) {
        float sum = lp0[i];
#pragma unroll
        for (int k = 0; k < 5; k++) {
          float m = (i - 1 - k >= 0) ? lp0[i - 1 - k] : 0.f;
          sum = sum + num[k] * m;
        }
        lp[i] = sum;
      }
    }
  MPHASE_END
  // -- second 2x decimation (pitch.c:305-308); the same lanes also form d[i] = y4[i+240]^2 - y4[i]^2,
  //    the increments of find_best_pitch's running energy (pitch.c:99)
  MPHASE_BEGIN
    if (a[q].ring) {
      const float *lp = PSM(q) + SM_LP;
      float *x4 = PSM(q) + SM_X4, *y4 = PSM(q) + SM_Y4, *syy = PSM(q) + SM_SYY;
      for (int j = t; j < 240; j += PITCH_THREADS) x4[j] = lp[384 + 2 * j];
      for (int j = t; j < 388; j += PITCH_THREADS) y4[j] = j < 387 ? lp[2 * j] : 0.f;
      for (int i = t; i < 147; i += PITCH_THREADS) {
        float hi = lp[2 * (i + 240)], lo = lp[2 * i];
        syy[i] = hi * hi - lo * lo;
      }
    }
  MPHASE_END
  // -- coarse search: 147 lags x 240 (rnn_pitch_xcorr pitch.c:216; each lag summed in order) on 30
  //    lanes x 5 lags of each stream's first warp, sliding register window; the running-energy chains
  //    of all streams share the lanes 0..NS-1 of one other warp.
  MPHASE_BEGIN
    if (t < 30 && a[q].ring) {
      const float *x4 = PSM(q) + SM_X4, *y4 = PSM(q) + SM_Y4;
      float *xc = PSM(q) + SM_XC;
      const float *yb = y4 + 5 * t;
      float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
      float w[5];
#pragma unroll
      for (int c = 0; c < 5; c++) w[c] = yb[c];
      for (int j0 = 0; j0 < 240; j0 += 5) {
#pragma unroll
        for (int r = 0; r < 5; r++) {
          const float xv = x4[j0 + r];
#pragma unroll
          for (int c = 0; c < 5; c++) acc[c] = acc[c] + xv * w[(c + r) % 5];
          const int nx = 5 * t + j0 + r + 5;
          w[r] = nx < 388 ? y4[nx] : 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < 5; c++) if (5 * t + c < 147) xc[5 * t + c] = acc[c];
    } else if (tid >= 32 && tid < 32 + PITCH_NS && a[tid - 32].ring) {
      float *sq = PSM(tid - 32);
      syy_running_inplace(sq + SM_SYY, sq_prefix(1.f, sq + SM_Y4, 240), 147);
    }
  MPHASE_END
  MPHASE_BEGIN
    if (tid < PITCH_NS && a[tid].ring) {
      float *sq = PSM(tid);
      int *mi = (int *)(sq + SM_PITCH_END + MI_INT);
      Best2 b2; best2_init(b2);
      for (int i0 = 0; i0 < 147; i0 += 3) {   // 147 = 49 * 3: a block's inputs loaded together, then visited in order, branch-free
        float xc3[3], sy3[3];                  // (32 registers per thread in this kernel: small blocks)
#pragma unroll
        for (int u = 0; u < 3; u++) { xc3[u] = sq[SM_XC + i0 + u]; sy3[u] = sq[SM_SYY + i0 + u]; }
#pragma unroll
        for (int u = 0; u < 3; u++) best2_visit_sel(b2, i0 + u, xc3[u], sy3[u]);
      }
      mi[0] = b2.p0; mi[1] = b2.p1;
    }
  MPHASE_END
  // -- xcorr := 0 (pitch.c:347) and the fine-stage increments d[i] = y[i+480]^2 - y[i]^2
  MPHASE_BEGIN
    if (a[q].ring) {
      const float *lp = PSM(q) + SM_LP;
      float *xc = PSM(q) + SM_XC, *syy = PSM(q) + SM_SYY;
      for (int i = t; i < 294; i += PITCH_THREADS) {
        xc[i] = 0.f;
        float hi = lp[i + 480], lo = lp[i];
        syy[i] = hi * hi - lo * lo;
      }
    }
  MPHASE_END
  // -- fine search around the two coarse winners (pitch.c:344-361): 10 lanes per stream packed from
  //    lane 0 on; the energy chains of all streams in the lanes of another warp
  MPHASE_BEGIN
    if (tid < 10 * PITCH_NS && a[tid / 10].ring) {
      const int qq = tid / 10, c = tid % 10;
      float *sq = PSM(qq);
      const int *mi = (const int *)(sq + SM_PITCH_END + MI_INT);
      const int c0 = 2 * mi[0], c1 = 2 * mi[1];
      int i = c < 5 ? c0 - 2 + c : c1 - 2 + (c - 5);
      bool ok = i >= 0 && i < 294;
      if (c >= 5) { int d = i - c0; if (d < 0) d = -d; if (d <= 2) ok = false; }
      if (ok) {
        const float *xl = sq + SM_LP + 384, *y = sq + SM_LP + i;
#if PITCH_CHAIN4
        const float sum = dot_chain4(0.f, xl, y, 480);
#else
        float sum = 0.f;
#pragma unroll 8
        for (int j = 0; j < 480; j++) sum = sum + xl[j] * y[j];
#endif
        sq[SM_XC + i] = RMAX(-1, sum);
      }
    } else if (tid >= 64 && tid < 64 + PITCH_NS && a[tid - 64].ring) {
      float *sq = PSM(tid - 64);
      syy_running_inplace(sq + SM_SYY, sq_prefix(1.f, sq + SM_LP, 480), 294);
    }
  MPHASE_END
  // -- pick the winner, pseudo-interpolate (pitch.c:362-384), enter the half-rate domain.  Only lags
  //    with xcorr > 0 can change find_best_pitch's state, and only the <= 10 searched lags are non-zero:
  //    visit those in ascending order.  Each stream's other warps meanwhile square the samples the
  //    yy_lookup chain of rnn_remove_doubling will need (pitch.c:454): a[i-1] = x[-i]^2, yyl[i] := x[N-i]^2.
  MPHASE_BEGIN
    if (tid < PITCH_NS && a[tid].ring) {
      float *sq = PSM(tid);
      const float *xc = sq + SM_XC, *syy = sq + SM_SYY;
      int *mi = (int *)(sq + SM_PITCH_END + MI_INT);
      const int c0 = 2 * mi[0], c1 = 2 * mi[1];
      const int lo = c0 < c1 ? c0 : c1, hi = c0 < c1 ? c1 : c0;
      Best2 b2; best2_init(b2);
      for (int i = lo - 2; i <= lo + 2; i++) if (i >= 0 && i < 294) best2_visit_sel(b2, i, xc[i], syy[i]);
      for (int i = hi - 2; i <= hi + 2; i++) if (i > lo + 2 && i >= 0 && i < 294) best2_visit_sel(b2, i, xc[i], syy[i]);
      int offset = 0;
      if (b2.p0 > 0 && b2.p0 < 293) {
        float aa = xc[b2.p0 - 1], bb = xc[b2.p0], cc = xc[b2.p0 + 1];
        if ((cc - aa) > .7f * (bb - aa)) offset = 1;
        else if ((aa - cc) > .7f * (bb - cc)) offset = -1;
      }
      int pitch_index = PITCH_MAX_PERIOD - (2 * b2.p0 - offset);      // denoise.c:365
      int T0 = pitch_index / 2;                                       // pitch.c:441
      if (T0 >= PITCH_MAX_PERIOD / 2) T0 = PITCH_MAX_PERIOD / 2 - 1;  // :445-446
      mi[4] = T0;
    }
    if (t >= 32 && a[q].ring) {
      float *sq = PSM(q);
      const float *x = sq + SM_LP + PITCH_MAX_PERIOD / 2;
      for (int i = 1 + (t - 32); i <= PITCH_MAX_PERIOD / 2; i += PITCH_THREADS - 32) {
        float u = x[-i], v = x[PITCH_FRAME_SIZE / 2 - i];
        sq[SM_X4 + i - 1] = u * u;   // x4/y4 are dead after the coarse search: 384 floats fit in their 628
        sq[SM_YYL + i] = v * v;
      }
    }
  MPHASE_END
  // -- all dot products rnn_remove_doubling can need, in parallel lanes (each one sequential):
  //    stream warp 0: xx, xy(T0), and xy(T1), xy(T1b) for k = 2..15      (pitch.c:449, 482)
  //    stream warp 1: speculative refinement lags T-1, T+1 of every candidate (pitch.c:513-514)
  //    lanes 64..64+NS-1 of the CTA: the yy_lookup energy chains of all streams (pitch.c:450-456)
  MPHASE_BEGIN
    const int N = PITCH_FRAME_SIZE / 2;
    if (tid >= 64 && tid < 64 + PITCH_NS) {
      if (a[tid - 64].ring) {
        float *sq = PSM(tid - 64);
        const float *x = sq + SM_LP + PITCH_MAX_PERIOD / 2;
        float *yyl = sq + SM_YYL;
        float yy = sq_prefix(0.f, x, N);   // == xx, summed in the same order (pitch.c:449-451)
        yyl[0] = yy;
        const float *a2 = sq + SM_X4;      // a2[i-1] = x[-i]^2, yyl[i] holds x[N-i]^2 until overwritten
        for (int i = 1; i <= PITCH_MAX_PERIOD / 2; i += 4) {
          f4 av = *(const f4 *)(a2 + i - 1);
          yy = yy + av.x - yyl[i];     yyl[i] = RMAX(0, yy);
          yy = yy + av.y - yyl[i + 1]; yyl[i + 1] = RMAX(0, yy);
          yy = yy + av.z - yyl[i + 2]; yyl[i + 2] = RMAX(0, yy);
          yy = yy + av.w - yyl[i + 3]; yyl[i + 3] = RMAX(0, yy);
        }
      }
    } else if (a[q].ring) {
      float *sq = PSM(q);
      const float *x = sq + SM_LP + PITCH_MAX_PERIOD / 2;
      float *dot = sq + SM_DOT;
      const int T0 = ((const int *)(sq + SM_PITCH_END + MI_INT))[4];
      if (t < 30) {
        int off, ok = 1;
        if (t == 0) off = 0;
        else if (t == 1) off = T0;
        else {
          int k = 2 + (t - 2) / 2, T1, T1b;
          rd_candidate(k, T0, &T1, &T1b);
          ok = T1 >= PITCH_MIN_PERIOD / 2;
          off = ((t - 2) & 1) ? T1b : T1;
        }
        if (ok) {
#if PITCH_CHAIN4
          dot[t] = dot_chain4(0.f, x, x - off, N);
#else
          float s = 0.f;
#pragma unroll 8
          for (int i = 0; i < N; i++) s = s + x[i] * x[i - off];
          dot[t] = s;
#endif
        }
      }
    }
  MPHASE_END
  // -- every candidate's pitch gain (pitch.c:458, 483-485: a double-precision sqrt and division each) is independent
  //    of the others: one lane per (stream, k), k = 1 (the initial candidate T0) .. 15; results in the dead xcorr array
  MPHASE_BEGIN
    if (tid < 15 * PITCH_NS && a[tid % PITCH_NS].ring) {
      const int qq = tid % PITCH_NS, k = 1 + tid / PITCH_NS;
      float *sq = PSM(qq);
      const float *dot = sq + SM_DOT, *yyl = sq + SM_YYL;
      const int T0 = ((const int *)(sq + SM_PITCH_END + MI_INT))[4];
      int T1, T1b;
      rd_candidate(k, T0, &T1, &T1b);
      if (k == 1 || T1 >= PITCH_MIN_PERIOD / 2) {
        const float xy = k == 1 ? dot[1] : .5f * (dot[2 + 2 * (k - 2)] + dot[3 + 2 * (k - 2)]);
        const float yy = k == 1 ? yyl[T0] : .5f * (yyl[T1] + yyl[T1b]);
        sq[SM_XC + k] = pitch_gain(xy, dot[0], yy);
        sq[SM_XC + 16 + k] = xy;
        sq[SM_XC + 32 + k] = yy;
      }
    }
  MPHASE_END
  // -- decision logic of rnn_remove_doubling (pitch.c:457-510) over the precomputed gains.  An accepted candidate only
  //    overwrites the running best and no threshold depends on an earlier acceptance, so walking k upwards with the
  //    gains at hand is the reference's loop.
  MPHASE_BEGIN
    if (tid < PITCH_NS && a[tid].ring) {
      const PitchArgs A = a[tid];
      float *sq = PSM(tid);
      const float *cg = sq + SM_XC, *cxy = sq + SM_XC + 16, *cyy = sq + SM_XC + 32;
      int *mi = (int *)(sq + SM_PITCH_END + MI_INT);
      const int T0 = mi[4], minperiod = PITCH_MIN_PERIOD / 2;
      int prev_period = ((const int *)A.pitch_state)[0] / 2;
      const float prev_gain = A.pitch_state[1];
      float best_xy = cxy[1], best_yy = cyy[1];
      const float g0 = cg[1];
      float g = g0;
      int Tb = T0, kbest = 1;
      for (int k = 2; k <= 15; k++) {
        int T1, T1b;
        rd_candidate(k, T0, &T1, &T1b);
        if (T1 < minperiod) break;
        const float g1 = cg[k];
        int d = T1 - prev_period; if (d < 0) d = -d;
        float cont;
        if (d <= 1) cont = prev_gain;
        else if (d <= 2 && 5 * k * k < T0) cont = .5f * prev_gain;
        else cont = 0;
        float thresh = RMAX(.3f, .7f * g0 - cont);
        if (T1 < 3 * minperiod) thresh = RMAX(.4f, .85f * g0 - cont);
        else if (T1 < 2 * minperiod) thresh = RMAX(.5f, .9f * g0 - cont);
        if (g1 > thresh) { best_xy = cxy[k]; best_yy = cyy[k]; Tb = T1; g = g1; kbest = k; }
      }
      best_xy = RMAX(0, best_xy);
      float pg;
      if (best_yy <= best_xy) pg = 1.f;
      else pg = best_xy / (best_yy + 1);
      if (pg > g) pg = g;
      mi[5] = Tb; mi[6] = kbest;
      sq[SM_PITCH_END + MI_AC] = pg;   // the autocorrelation slots are long dead
    }
  MPHASE_END
  // -- the two refinement correlations around the chosen period (pitch.c:513-514: xcorr[k] = <x, x-(T+k-1)>, k = 0, 2;
  //    the centre lag was summed with the candidates in the same order) -- 2 instead of 30 speculative ones
  MPHASE_BEGIN
    if (tid < 2 * PITCH_NS && a[tid % PITCH_NS].ring) {
      const int qq = tid % PITCH_NS, side = tid / PITCH_NS;
      float *sq = PSM(qq);
      const float *x = sq + SM_LP + PITCH_MAX_PERIOD / 2;
      const int Tb = ((const int *)(sq + SM_PITCH_END + MI_INT))[5];
      const int off = side ? Tb + 1 : Tb - 1;
#if PITCH_CHAIN4
      sq[SM_DOT + 32 + side] = dot_chain4(0.f, x, x - off, PITCH_FRAME_SIZE / 2);
#else
      float s2 = 0.f;
#pragma unroll 8
      for (int i = 0; i < PITCH_FRAME_SIZE / 2; i++) s2 = s2 + x[i] * x[i - off];
      sq[SM_DOT + 32 + side] = s2;
#endif
    }
  MPHASE_END
  // -- final offset (pitch.c:515-524) + state update (denoise.c:369-370)
  MPHASE_BEGIN
    if (tid < PITCH_NS && a[tid].ring) {
      const PitchArgs A = a[tid];
      float *sq = PSM(tid);
      const float *dot = sq + SM_DOT;
      int *mi = (int *)(sq + SM_PITCH_END + MI_INT);
      const int Tb = mi[5], kbest = mi[6];
      const float xc0 = dot[32], xc2 = dot[33];
      const float xc1 = kbest == 1 ? dot[1] : dot[2 + 2 * (kbest - 2)];
      int offset;
      if ((xc2 - xc0) > .7f * (xc1 - xc0)) offset = 1;
      else if ((xc0 - xc2) > .7f * (xc1 - xc2)) offset = -1;
      else offset = 0;
      int Tout = 2 * Tb + offset;
      if (Tout < PITCH_MIN_PERIOD) Tout = PITCH_MIN_PERIOD;
      mi[2] = Tout;
      ((int *)A.pitch_state)[0] = Tout;
      A.pitch_state[1] = sq[SM_PITCH_END + MI_AC];
    }
  MPHASE_END
}

// Spectral half of rnn_compute_frame_features (src/denoise.c:358, 371-397) incl. rnn_frame_analysis
// (:332-345): X, P, band energies / correlation, log-energy features, silence test.
// TRAIN selects the reference's -DTRAINING=1 semantics (the build src/dump_features.c uses): X is
// low-passed at a.lowpass (:340-343), a quiet frame does NOT short-circuit the features (:389) and the
// returned flag is E < 0.1 (:397).
template <bool TRAIN>
HD void spectrum_stream(float *sm, const SpectrumArgs a, const DspTables *T) {
  float *misc = sm + SM_SPEC_END;
  int *mi = (int *)(misc + SMI_INT);
  cpx *F = (cpx *)(sm + SM_F), *XS = (cpx *)(sm + SM_XS);
  float *win = sm + SM_WIN;
  const int pitch_T = ((const int *)a.pitch_state)[0];
  short *eb = (short *)(misc + SMI_EBAND);
  float *hws = sm + SM_XS;   // the half window, staged for the first transform (bins of X live here afterwards)
  // the pitch-lagged window starts at ring position q0 (any alignment): it is fetched as the 241 aligned 16-byte pieces
  // that cover it and read from `lag` floats into the staging buffer
  int q0 = a.ring_base + PITCH_BUF_SIZE - WINDOW_SIZE - pitch_T;
  if (q0 >= PITCH_BUF_SIZE) q0 -= PITCH_BUF_SIZE;
  if (q0 < 0) q0 += PITCH_BUF_SIZE;
  const int lag = q0 & 3;
  // -- X = FFT(window * [previous frame | this frame]) (denoise.c:332-339); the analysis window
  //    is the last 960 samples of the updated pitch history.
  PHASE_BEGIN
    // asynchronous 16-byte copies (ring base and window start are multiples of 4 floats; a piece never straddles the
    // ring's end), all of a thread's requests in flight together, L1 bypassed; the half window and the band edges
    // come along, so that stage 1 and the band sums read shared memory instead of waiting on the L2 for the tables
    static_assert(PITCH_BUF_SIZE % 4 == 0 && FRAME_SIZE % 4 == 0 && (PITCH_BUF_SIZE - WINDOW_SIZE) % 4 == 0, "aligned pieces");
    for (int c = tid; c < WINDOW_SIZE / 4; c += nthr) {
      int p = a.ring_base + PITCH_BUF_SIZE - WINDOW_SIZE + 4 * c; if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
      async_copy16(win + 4 * c, a.ring + p);
    }
    for (int c = tid; c < FRAME_SIZE / 4; c += nthr) async_copy16(hws + 4 * c, T->half_window + 4 * c);
    if (tid < (NB_BANDS + 2) / 2) async_copy4((float *)eb + tid, (const float *)T->eband + tid);
    async_wait_all();
  PHASE_END
  PHASE_BEGIN fft_stage1(F, win, nullptr, T, tid, nthr, hws); PHASE_END
  PHASE_BEGIN
    // the staging buffer is dead until the second transform: start fetching the pitch-lagged window
    // into it now (asynchronous copies), so the ring's latency hides behind the first transform
    for (int c = tid; c < WINDOW_SIZE / 4 + 1; c += nthr) {
      int p = q0 - lag + 4 * c; if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
      async_copy16(win + 4 * c, a.ring + p);
    }
    fft_radix4(F, 4, 16, 60, T, tid, nthr);
  PHASE_END
  PHASE_BEGIN fft_radix4(F, 16, 64, 15, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix3(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix5(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN
    for (int i = tid; i < FREQ_SIZE; i += nthr) {
      cpx v = F[fsw(i)];
      if (TRAIN && i >= a.lowpass) v.r = v.i = 0.f;
      if (i < 400) XS[i] = v;
      st_stream2(a.spec_out + 2 * i, v.r, v.i);
    }
    async_wait_all();   // the lagged window is in `win` once this phase's barrier is passed
  PHASE_END
  // -- P = FFT(window * pitch_buf[768-T .. 768-T+960)) (denoise.c:371-374)
  PHASE_BEGIN fft_stage1(F, win + lag, nullptr, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix4(F, 4, 16, 60, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix4(F, 16, 64, 15, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix3(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix5(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN
    cpx *PT = F + 512;   // |P|^2 terms: the upper half of the work buffer (bins 0..480 park below element 496)
    for (int i = tid; i < FREQ_SIZE; i += nthr) {
      cpx v = F[fsw(i)];
      st_stream2(a.spec_out + 2 * (FREQ_SIZE + i), v.r, v.i);
      if (i < 400) {
        // weighted per-bin terms of the three band sums (band_sum_pre): X's over the complex value they came from (this
        // thread's own slot), P's into the dead upper half of the work buffer, X.P's into the dead window staging; all
        // three as (frac term, 1 - frac term) pairs
        const cpx x = XS[i];
        const float wf = T->bin_frac[i], wc = T->bin_cfrac[i];
        const float tx = bin_term(x, x), tp = bin_term(v, v), txp = bin_term(x, v);
        XS[i].r = wf * tx; XS[i].i = wc * tx;
        PT[i].r = wf * tp; PT[i].i = wc * tp;
        win[2 * i] = wf * txp; win[2 * i + 1] = wc * txp;
      }
    }
  PHASE_END
  // -- the three sets of 34 triangular band sums (compute_band_energy / compute_band_corr), one lane each
  PHASE_BEGIN
    // Chain lengths run from 2 terms (band 0) to 83 (band 32) and a warp takes as long as its longest lane: the 102
    // chains are dealt to the lanes longest first (lane L: band 33 - L / 3, set L % 3), so that warp 0 holds the eleven
    // widest bands of all three sets and the other warps finish after 30, 8 and 4 steps -- 125 warp-steps instead of
    // 4 x 80 with the sets laid out one after the other (this phase was a fifth of the kernel's instructions).
    if (tid < 3 * (NB_BANDS + 2)) {
      // (the three sets' terms have the same interleaved layout -- frac term, 1 - frac term per bin -- so that the lanes of
      //  a warp, which hold all three sets, run ONE instruction stream; with a different layout for the X.P terms the sets
      //  were three divergent paths executed one after the other)
      const int b = NB_BANDS + 1 - tid / 3, set = tid % 3;
      const float *terms = set == 0 ? (const float *)XS : set == 1 ? (const float *)(F + 512) : (const float *)win;
      misc[SMI_BAND + 34 * set + b] = band_sum_pre(b, terms, 2, 1, eb);
    }
  PHASE_END
  // -- Ex, Ep, Exp (denoise.c:344,375-377)
  // (the FFT buffer is dead from here on: the 32 x 32 DCT table is fetched into it with asynchronous 16-byte copies --
  //  no thread waits for them before the follower phase -- so that the two DCTs at the end read shared memory
  //  instead of 32 dependent L1/L2 round trips)
  float *dct_sm = sm + SM_F;
  PHASE_BEGIN
    for (int c = tid; c < NB_BANDS * NB_BANDS / 4; c += nthr) async_copy16(dct_sm + 4 * c, T->dct + 4 * c);
    if (tid < NB_BANDS) {
      float ex = band_finish(misc + SMI_BAND, tid);
      float ep = band_finish(misc + SMI_BAND + 34, tid);
      float exp_ = band_finish(misc + SMI_BAND + 68, tid);
      exp_ = (float)(exp_ / sqrt(.001 + ex * ep));
      misc[SMI_E + tid] = ex; misc[SMI_E + 32 + tid] = ep; misc[SMI_E + 64 + tid] = exp_;
      a.band_out[tid] = ex; a.band_out[32 + tid] = ep; a.band_out[64 + tid] = exp_;
    }
  PHASE_END
  // -- log-energy floor follower + silence test (denoise.c:380-393): the 32 log10() are independent
  //    (one lane each); only the follower itself is a serial chain.
  PHASE_BEGIN
    if (tid < NB_BANDS) misc[SMI_LY + tid] = (float)log10(1e-2 + misc[SMI_E + tid]);
  PHASE_END
  PHASE_BEGIN
    if (tid == 0) {
      float logMax = -2, follow = -2;
      // The reference evaluates follow - 1.5 and both maxima in double and rounds on the stores to ly[i] and follow
      // (denoise.c:384-386).  follow - 1.5 is exact in double (24-bit operands a few binades apart), rounding is
      // monotonic -- float(max(a, b)) == max(float(a), float(b)) -- and the other operands are floats already, so the
      // same values come out of float arithmetic: follow - 1.5f is the single correct rounding of the exact
      // difference.  32 dependent steps of 3 float ops instead of conversions and FP64 ops on one thread
      // (tests/test_dsp_emulation.py holds this source against the literal double form).
      // The chain runs on registers: 16 inputs per 16-byte vector loads, 16 steps, 16 outputs per vector stores (one
      // shared-memory round trip per step made this phase 11 % of the CTA's lifetime).
#pragma unroll
      for (int hb = 0; hb < NB_BANDS; hb += 16) {
        f4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = *(const f4 *)(misc + SMI_LY + hb + 4 * u);
        float l[16] = {v[0].x, v[0].y, v[0].z, v[0].w, v[1].x, v[1].y, v[1].z, v[1].w,
                       v[2].x, v[2].y, v[2].z, v[2].w, v[3].x, v[3].y, v[3].z, v[3].w};
#pragma unroll
        for (int i = 0; i < 16; i++) {
          float ly = l[i];
          const float f15 = follow - 1.5f;
          const float m1 = RMAX(f15, ly);
          const float lm7 = logMax - 7;
          ly = RMAX(lm7, m1);
          logMax = RMAX(logMax, ly);
          follow = RMAX(f15, ly);
          l[i] = ly;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
          f4 o; o.x = l[4 * u]; o.y = l[4 * u + 1]; o.z = l[4 * u + 2]; o.w = l[4 * u + 3];
          *(f4 *)(misc + SMI_LY + hb + 4 * u) = o;
        }
      }
    } else if (tid == 32) {
      // the frame energy (denoise.c:387) is its own chain: a lane of another warp adds it beside the follower
      float E = 0;
      f4 v[8];
#pragma unroll
      for (int u = 0; u < 8; u++) v[u] = *(const f4 *)(misc + SMI_E + 4 * u);
#pragma unroll
      for (int u = 0; u < 8; u++) { E += v[u].x; E += v[u].y; E += v[u].z; E += v[u].w; }
      int silent = !TRAIN && E < 0.04;
      mi[3] = silent;
      a.silence[0] = TRAIN ? E < 0.1 : silent;
    }
    async_wait_all();   // the DCT table is in shared memory once this phase's barrier is passed
  PHASE_END
  // -- features (denoise.c:378-379, 391, 394-396)
  PHASE_BEGIN
    const int silent = mi[3];
    if (tid < NB_BANDS) {
      float v = dct_one_tab(misc + SMI_LY, tid, dct_sm);
      if (tid == 0) v -= 12;
      if (tid == 1) v -= 4;
      a.features[tid] = silent ? 0.f : v;
    } else if (tid < 2 * NB_BANDS) {
      float v = dct_one_tab(misc + SMI_E + 64, tid - NB_BANDS, dct_sm);
      a.features[tid] = silent ? 0.f : v;
    } else if (tid == 2 * NB_BANDS) {
      a.features[tid] = silent ? 0.f : (float)(.01 * (pitch_T - 300));
    }
  PHASE_END
}

// Training targets (the per-frame body of src/dump_features.c:466-491, a -DTRAINING=1 build): after
// spectrum_stream<true> of the noisy frame (features -> rec[0..65), Ex left in misc[SMI_E..]), analyse the
// clean frame (rnn_frame_analysis on the clean state: window, FFT, low-pass, band energies Ey) and derive
// the ideal band gains g = min(1, sqrt((Ey + 1e-3) / (Ex + 1e-3))), -1 where the target is undefined.
struct TrainArgs {
  const float *clean;   // [480] clean speech frame
  float *clean_mem;     // [480] previous clean frame (analysis_mem of the clean state)
  float *rec;           // [98]  features[65] | g[32] | vad target
  const int *quiet;     // [1]   flag written by spectrum_stream<true> (E < 0.1)
  int lowpass, band_lp; // the sequence's low-pass bin and the first band above it (dump_features.c:400-406)
  float vad_target;
  int noise_free;       // noise_gain == 0 && fgnoise_gain == 0 (dump_features.c:477)
};
HD void train_targets_stream(float *sm, const TrainArgs a, const DspTables *T) {
  float *misc = sm + SM_SPEC_END;
  cpx *F = (cpx *)(sm + SM_F);
  float *win = sm + SM_WIN;
  PHASE_BEGIN
    for (int i = tid; i < FRAME_SIZE; i += nthr) { win[i] = a.clean_mem[i]; win[FRAME_SIZE + i] = a.clean[i]; }
  PHASE_END
  PHASE_BEGIN
    for (int i = tid; i < FRAME_SIZE; i += nthr) a.clean_mem[i] = win[FRAME_SIZE + i];
    fft_stage1(F, win, nullptr, T, tid, nthr);
  PHASE_END
  PHASE_BEGIN fft_radix4(F, 4, 16, 60, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix4(F, 16, 64, 15, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix3(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix5(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN
    for (int i = tid; i < 400; i += nthr) {
      cpx v = F[fsw(i)];
      if (i >= a.lowpass) v.r = v.i = 0.f;
      const float ty = bin_term(v, v);
      win[i] = T->bin_frac[i] * ty; win[400 + i] = T->bin_cfrac[i] * ty;
    }
  PHASE_END
  PHASE_BEGIN
    if (tid < NB_BANDS + 2) misc[SMI_BAND + tid] = band_sum_pre(tid, win, 1, 400, T->eband);
  PHASE_END
  PHASE_BEGIN
    if (tid < NB_BANDS) {
      const float ey = band_finish(misc + SMI_BAND, tid), ex = misc[SMI_E + tid];
      float g = (float)sqrt((ey + 1e-3) / (ex + 1e-3));
      if (g > 1) g = 1;
      if (a.quiet[0] || tid > a.band_lp) g = -1;
      if (ey < 5e-2 && ex < 5e-2) g = -1;
      if (a.vad_target == 0 && a.noise_free) g = -1;
      a.rec[NB_FEATURES + tid] = g;
    } else if (tid == NB_BANDS) {
      a.rec[NB_FEATURES + NB_BANDS] = a.vad_target;
    }
  PHASE_END
}

struct SynthesisArgs {
  float *spec_delayed;      // [2][962] X and P of the PREVIOUS frame (modified in place, then dead)
  const float *band_delayed;// [3][32]  Ex, Ep, Exp of the previous frame
  const float *band_cur;    // [3][32]  Ex of this frame is [0..32)
  const float *gains;       // [32] network output of this frame
  const int *silence;       // [1]
  float *lastg;             // [32]
  float *synthesis_mem;     // [480]
  float *out;               // [480] float PCM, or
  short *out_s16;           // [480] 16-bit PCM (non-null selects it): the C cast of examples/rnnoise_demo.c:58
};

// shared-memory plan of the synthesis CTA (floats)
#define SS_X 0                        // [962] delayed X
#define SS_P (SS_X + 2 * FREQ_SIZE)   // [800] bins 0..399 of the delayed P (the pitch filter's gain is 0 from bin 400 on); once P is dead,
                                      //       the overlap memory is prefetched into its place
#define SS_F (SS_P + 2 * 400)         // [1920] FFT buffer
#define SS_V (SS_F + 2 * WINDOW_SIZE) // [6][34] band vectors: r, norm, g, sums...
#define SS_TOTAL (SS_V + 6 * 34)
// 3886 floats: 14 CTAs per SM (13 with all 481 bins of P resident).  Prefetching the synthesis window next to the overlap memory would need 960
// floats there and cost that 14th CTA; the window is a table every CTA reads (L1 / L2 hits).
static_assert((SS_TOTAL * 4 + 1024) * 14 <= 228 * 1024, "synthesis kernel: 14 CTAs per SM");

// rnn_pitch_filter (denoise.c:421-455), gain smoothing + interpolation (:479-493),
// frame_synthesis (:400-407) with inverse_transform (:200-217).
HD void synthesis_stream(float *sm, const SynthesisArgs a, const DspTables *T) {
  cpx *X = (cpx *)(sm + SS_X), *P = (cpx *)(sm + SS_P), *F = (cpx *)(sm + SS_F);
  float *r = sm + SS_V, *sums = sm + SS_V + 34, *norm = sm + SS_V + 68, *g = sm + SS_V + 102;
  const int silent = a.silence[0];
  PHASE_BEGIN
    // X (all bins) and bins 0..399 of P arrive by asynchronous copies, all of a thread's requests in flight together:
    // 16-byte pieces (L1 bypassed) for bins 0..399 of X and bins 1..400 of P -- floats [0, 800) and [964, 1764) of the
    // spectrum slot, which is laid out exactly like SS_X | SS_P (the last piece's second half, P bin 400, lands on the
    // idle FFT buffer) -- and 8-byte pieces for the 81 tail bins of X and bin 0 of P.
    // The pitch filter's gain is 0 from bin 400 on (interp_band_gain leaves those bins at 0, denoise.c:140-154,
    // 432-438): their update x += 0 * p is done here by the thread that fetched the bin, with P's tail in registers, so
    // that it need not stay resident -- the same multiply and add as in the filter phase below.
    static_assert(FREQ_SIZE - 400 < DSP_THREADS, "one tail bin per thread, one more thread for bin 0 of P");
    static_assert(SS_P == 2 * FREQ_SIZE && (SS_P + 2) % 4 == 0, "slot layout == shared layout; P bin 1 is 16-byte aligned");
    for (int c = tid; c < 200; c += nthr) {
      async_copy16(sm + SS_X + 4 * c, a.spec_delayed + 4 * c);
      async_copy16(sm + SS_P + 2 + 4 * c, a.spec_delayed + SS_P + 2 + 4 * c);
    }
    int itail = -1;
    cpx ptail; ptail.r = ptail.i = 0.f;
    if (tid < FREQ_SIZE - 400) {
      const int i = 400 + tid;
      async_copy8(&X[i], a.spec_delayed + 2 * i);
      if (!silent) {
        itail = i;
        ptail.r = ld_stream(a.spec_delayed + 2 * (FREQ_SIZE + i)); ptail.i = ld_stream(a.spec_delayed + 2 * (FREQ_SIZE + i) + 1);
      }
    } else if (tid == FREQ_SIZE - 400) {
      async_copy8(&P[0], a.spec_delayed + 2 * FREQ_SIZE);
    }
    if (!silent && tid < NB_BANDS) {
      const float Ex = a.band_delayed[tid], Ep = a.band_delayed[32 + tid], Exp = a.band_delayed[64 + tid];
      const float gg = a.gains[tid];
      float rr;
      if (Exp > gg) rr = 1;
      else {
        float e2 = Exp * Exp, g2 = gg * gg;
        rr = (float)((e2 * (1 - g2)) / (.001 + g2 * (1 - e2)));
      }
      float c = RMAX(0, rr);
      c = RMIN(1, c);
      rr = (float)sqrt((double)c);
      rr = (float)(rr * sqrt(Ex / (1e-8 + Ep)));
      r[tid] = rr;
    }
    async_wait_all();   // a thread sees its own copies: the tail bin below was fetched by this thread
    if (itail >= 0) {
      cpx x = X[itail];
      x.r += 0.f * ptail.r;
      x.i += 0.f * ptail.i;
      X[itail] = x;
    }
  PHASE_END
  if (!silent) {
    PHASE_BEGIN
      for (int i = tid; i < 400; i += nthr) {   // bins 400..480: done at load time
        float rf = interp_bin(r, i, T);
        cpx x = X[i], p = P[i];
        x.r += rf * p.r;
        x.i += rf * p.i;
        X[i] = x;
        // weighted band-sum terms into the (still idle) FFT buffer
        const float tx = bin_term(x, x);
        sm[SS_F + i] = T->bin_frac[i] * tx; sm[SS_F + 400 + i] = T->bin_cfrac[i] * tx;
      }
    PHASE_END
    PHASE_BEGIN
        if (tid < NB_BANDS + 2) sums[tid] = band_sum_pre(tid, sm + SS_F, 1, 400, T->eband);
    PHASE_END
    PHASE_BEGIN
        if (tid < NB_BANDS) {
        float newE = band_finish(sums, tid);
        norm[tid] = (float)sqrt(a.band_delayed[tid] / (1e-8 + newE));
        // gain smoothing (denoise.c:479-487)
        float gg = a.gains[tid];
        float lg = a.lastg[tid];
        float al = .6f * lg;
        gg = RMAX(gg, al);
        double t = gg * (a.band_delayed[tid] + 1e-3) / (a.band_cur[tid] + 1e-3);
        a.lastg[tid] = (float)RMIN(1.f, t);
        g[tid] = gg;
      }
    PHASE_END
    PHASE_BEGIN
      for (int i = tid; i < FREQ_SIZE; i += nthr) {
        float nf = interp_bin(norm, i, T);
        float gf = interp_bin(g, i, T);
        cpx x = X[i];
        x.r *= nf; x.i *= nf;
        x.r *= gf; x.i *= gf;
        X[i] = x;
      }
    PHASE_END
  }
  // P is dead once the pitch filter has run: fetch the overlap memory into its place with asynchronous copies now, and --
  // X being dead once stage 1 has gathered it -- the synthesis window into X's place during the next phase, so that the
  // output phase waits neither on HBM nor on the L2 for them (it was 30 % of this CTA's lifetime: four dependent
  // round trips per thread for the window)
  float *ola = sm + SS_P + 2;   // 16-byte aligned
  float *hws = sm + SS_X;
  PHASE_BEGIN
    for (int c = tid; c < FRAME_SIZE / 4; c += nthr) async_copy16(ola + 4 * c, a.synthesis_mem + 4 * c);
    fft_stage1(F, nullptr, X, T, tid, nthr);
  PHASE_END
  PHASE_BEGIN
    for (int c = tid; c < FRAME_SIZE / 4; c += nthr) async_copy16(hws + 4 * c, T->half_window + 4 * c);
    fft_radix4(F, 4, 16, 60, T, tid, nthr);
  PHASE_END
  PHASE_BEGIN fft_radix4(F, 16, 64, 15, T, tid, nthr); PHASE_END
  PHASE_BEGIN fft_radix3(F, T, tid, nthr); PHASE_END
  PHASE_BEGIN
    fft_radix5(F, T, tid, nthr);
    async_wait_all();   // overlap memory + window are in shared memory once this phase's barrier is passed
  PHASE_END
  PHASE_BEGIN
    // t[i] = 960 * y[(960 - i) % 960].re, windowed; out = first half + overlap memory.  A thread's operands are
    // loaded for all of its samples first, then combined
    // (two samples at a time: the kernel keeps 14 CTAs per SM with 36 registers per thread)
    constexpr int NI = (FRAME_SIZE + DSP_THREADS - 1) / DSP_THREADS;
    static_assert(NI % 2 == 0, "pairs");
#pragma unroll
    for (int u0 = 0; u0 < NI; u0 += 2) {
      float y0[2], y1[2], w0[2], w1[2], ol[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int i = tid + (u0 + u) * DSP_THREADS, ii = i < FRAME_SIZE ? i : 0;
        y0[u] = F[fsw(ii ? WINDOW_SIZE - ii : 0)].r;
        y1[u] = F[fsw(WINDOW_SIZE - (FRAME_SIZE + ii))].r;   // index 480+i -> y[480-i]
        w0[u] = hws[ii];
        w1[u] = hws[FRAME_SIZE - 1 - ii];
        ol[u] = ola[ii];
      }
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int i = tid + (u0 + u) * DSP_THREADS;
        if (i < FRAME_SIZE) {
          float t0 = WINDOW_SIZE * y0[u];
          float t1 = WINDOW_SIZE * y1[u];
          t0 *= w0[u];
          t1 *= w1[u];
          const float o = t0 + ol[u];
          if (a.out_s16) a.out_s16[i] = (short)(int)o;   // truncation toward zero, low 16 bits (x86 cvttss2si + narrowing)
          else st_stream(a.out + i, o);
          st_stream(a.synthesis_mem + i, t1);
        }
      }
    }
  PHASE_END
}
