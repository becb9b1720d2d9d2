// dsp_pitch.cuh -- pitch half of rnn_compute_frame_features (src/denoise.c:359-370):
// rnn_pitch_downsample / rnn_pitch_search / rnn_remove_doubling (src/pitch.c:146,281,423) for a GROUP of
// PG streams per CTA (the default pitch kernel; pitch_streams in dsp_stream.cuh is the round-1 kernel, kept
// as a cross-check that runs the same arithmetic under another thread mapping).
//
// Execution model.  The pitch analysis is a chain of phases that are either WIDE (element-parallel over a
// stream's 864 half-rate samples, or 30 independent dot products per stream) or NARROW (a handful of serial
// float chains per stream: 5 autocorrelation lags, 3 running energies, 10 fine-search lags, the selection
// scans, the final decision).  Bit-exact parity with the reference forbids splitting any of those sums, so
// the only way to keep lanes busy is to put the SAME chain of DIFFERENT streams side by side:
//   * warp q < PG is the home warp of stream q: all wide work of that stream (lanes = samples / lags);
//   * narrow work is laid out stream-minor over the first lanes of the CTA: lane l -> (stream l % PG,
//     chain l / PG), so one warp runs the same chain for 16+ streams with every lane busy;
//   * three extra warps run the three running-energy chains (find_best_pitch's Syy at both rates and
//     rnn_remove_doubling's yy_lookup), lane = stream, CONCURRENTLY with the coarse correlation -- they only
//     depend on the whitened signal -- so they never sit on the critical path.
// Against the round-1 mapping (4 streams x 96 threads, narrow phases packed 4 wide) this executes ~40 % fewer
// warp instructions per stream and replaces the 30 speculative refinement dot products of
// rnn_remove_doubling by the 2 that are needed, computed after the decision (pitch.c:513-514).
// Shared memory: one padded row of P2_STRIDE floats per stream (odd stride: lane = stream accesses of one
// element index fall into 16 different banks).
#pragma once
#include "dsp_core.cuh"

#ifndef PG
#define PG 16                      // streams per CTA
#endif
#define PG_CHAIN_WARPS 3
#define PG_WARPS (PG + PG_CHAIN_WARPS)
#define PG_THREADS (32 * PG_WARPS)
static_assert(PG >= 4 && PG <= 29 && 10 * PG <= PG_THREADS, "narrow phases are laid out over the first 10 * PG threads");

// per-stream shared-memory row (floats)
#define P2_LP 0                      // [864] whitened half-rate signal x_lp
#define P2_B (P2_LP + LP_SIZE)       // [864] lp0 until the FIR | x4[240] y4[388] (coarse) | xc2[296] (fine)
#define P2_X4 P2_B
#define P2_Y4 (P2_B + 240)
#define P2_XC2 P2_B
#define P2_XC4 (P2_B + LP_SIZE)      // [148] coarse correlations; after the coarse scan: candidate gains / xy / yy [3][16]
#define P2_CAND P2_XC4
#define P2_SYY4 (P2_XC4 + 148)       // [148] running energy seen by the coarse scan
#define P2_SYY2 (P2_SYY4 + 148)      // [296] running energy seen by the fine scan
#define P2_YYL (P2_SYY2 + 296)       // [388] yy_lookup
#define P2_DOT (P2_YYL + 388)        // [64]  remove_doubling dot products
#define P2_MISC (P2_DOT + 64)        // [32]  ac[5] @0, taps[5] @8, ints @16, floats @24
#define P2_STRIDE (P2_MISC + 32 + 1) // odd
static_assert(P2_STRIDE % 2 == 1, "odd row stride");
#define PM_AC 0
#define PM_NUM 8
#define PM_INT 16    // [0] best0 [1] best1 [2] T0 (half rate) [3] Tb [4] kbest
#define PM_F 24      // [0] pg (already limited by g)

struct PitchGroup {
  const float *xb;      // [n][480]  frames of this group's streams after the high-pass biquad
  float *ring;          // [n][1728] pitch-history rings
  float *pitch_state;   // [n][2]    {last_period as int bits, last_gain}: read as the prior, then updated
  int n;                // live streams of this group (1..PG)
  int ring_base;        // physical index of logical sample 0 AFTER this frame's 480-sample shift
};

#if defined(__CUDACC__) && defined(PITCH_TIMING)
// diagnostics build (-DPITCH_TIMING=<cta>): that CTA's thread 0 records clock64() after every phase barrier
__device__ long long g_pitch_t[32];
#endif
#if defined(__CUDA_ARCH__) && defined(PITCH_TIMING)
#define GPHASE_BEGIN { const int tid = threadIdx.x; const int w = tid >> 5, ln = tid & 31; (void)w; (void)ln;
#define GPHASE_END } __syncthreads(); if (blockIdx.x == PITCH_TIMING && threadIdx.x == 0 && phase_no < 32) g_pitch_t[phase_no] = clock64(); phase_no++;
#elif defined(__CUDA_ARCH__)
#define GPHASE_BEGIN { const int tid = threadIdx.x; const int w = tid >> 5, ln = tid & 31; (void)w; (void)ln;
#define GPHASE_END } __syncthreads();
#else
#define GPHASE_BEGIN for (int tid = 0; tid < PG_THREADS; ++tid) { const int w = tid >> 5, ln = tid & 31; (void)w; (void)ln;
#define GPHASE_END }
#endif
#define GSM(q) (sm + (q) * P2_STRIDE)

// One serial dot product <x[0..n), y[0..n)>, summed in index order (xcorr_kernel / celt_inner_prod order).
// The chain of n dependent additions is the critical path of the narrow phases, and a single warp does not hide
// its own shared-memory latency: the operands are fetched in register blocks of 8, the next block's loads issued
// before the current block's additions.
HD float dot_seq(const float *x, const float *y, int n) {
  float s = 0.f;
  const int nb = n & ~7;
  float a[8], b[8];
  if (nb) {
#pragma unroll
    for (int t = 0; t < 8; t++) { a[t] = x[t]; b[t] = y[t]; }
  }
  for (int i = 0; i < nb; i += 8) {
    float na[8], nb2[8];
    const bool more = i + 8 < nb;
    if (more) {
#pragma unroll
      for (int t = 0; t < 8; t++) { na[t] = x[i + 8 + t]; nb2[t] = y[i + 8 + t]; }
    }
#pragma unroll
    for (int t = 0; t < 8; t++) s = s + a[t] * b[t];
    if (more) {
#pragma unroll
      for (int t = 0; t < 8; t++) { a[t] = na[t]; b[t] = nb2[t]; }
    }
  }
  for (int i = nb; i < n; i++) s = s + x[i] * y[i];
  return s;
}

HD void pitch_group(float *sm, const PitchGroup g) {
  const int H = PITCH_BUF_SIZE - FRAME_SIZE;
#if defined(__CUDA_ARCH__) && defined(PITCH_TIMING)
  int phase_no = 1;
  if (blockIdx.x == PITCH_TIMING && threadIdx.x == 0) g_pitch_t[0] = clock64();
#endif
  // -- P1: append the new frame to the history ring (denoise.c:359-360; a ring instead of the memmove) and
  //    decimate by 2 straight from HBM/L2 (pitch.c:171-173).  The 480 ring slots being overwritten hold the
  //    oldest samples, which the decimation never reads.
  GPHASE_BEGIN
    if (w < g.n) {
      const float *xb = g.xb + (size_t)w * FRAME_SIZE;
      float *ring = g.ring + (size_t)w * PITCH_BUF_SIZE;
      float *lp0 = GSM(w) + P2_B;
      // global loads in batches of independent requests (a warp walks its stream alone: without the batching the
      // 27 + 15 round trips to L2 / HBM were 19 k cycles of the phase)
      {
        float v[15];
#pragma unroll
        for (int u = 0; u < 15; u++) v[u] = xb[ln + 32 * u];
#pragma unroll
        for (int u = 0; u < 15; u++) {
          int p = g.ring_base + H + ln + 32 * u; if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
          ring[p] = v[u];
        }
      }
#pragma unroll
      for (int b0 = 0; b0 < 27; b0 += 9) {
        float c[9], r[9], l[9];
#pragma unroll
        for (int u = 0; u < 9; u++) {
          const int i = ln + 32 * (b0 + u), k = 2 * i;
          c[u] = k < H ? ring_at(ring, g.ring_base, k) : xb[k - H];
          r[u] = k + 1 < H ? ring_at(ring, g.ring_base, k + 1) : xb[k + 1 - H];
          l[u] = i == 0 ? 0.f : k - 1 < H ? ring_at(ring, g.ring_base, k - 1) : xb[k - 1 - H];
        }
#pragma unroll
        for (int u = 0; u < 9; u++) {
          const int i = ln + 32 * (b0 + u);
          lp0[i] = i ? .5f * (.5f * (l[u] + r[u]) + c[u]) : .5f * (.5f * r[u] + c[u]);
        }
      }
    }
  GPHASE_END
  // -- P2: autocorrelation lags 0..4 (celt_lpc.c:92-174: first n-4 samples, then the tail)
  GPHASE_BEGIN
    if (tid < 5 * PG && tid % PG < g.n) {
      const int q = tid % PG, k = tid / PG, fastN = LP_SIZE - 4;
      const float *lp0 = GSM(q) + P2_B;
      const float s = dot_seq(lp0, lp0 + k, fastN);
      float d = 0.f;
      for (int i = k + fastN; i < LP_SIZE; i++) d = d + lp0[i] * lp0[i - k];
      GSM(q)[P2_MISC + PM_AC + k] = s + d;
    }
  GPHASE_END
  // -- P3: LPC -> whitening taps (pitch.c:181-212, celt_lpc.c:38-89)
  GPHASE_BEGIN
    if (tid < g.n) lpc_taps(GSM(tid) + P2_MISC + PM_AC, GSM(tid) + P2_MISC + PM_NUM);
  GPHASE_END
  // -- P4: 5-tap whitening FIR with zero history (celt_fir5, pitch.c:104-143)
  GPHASE_BEGIN
    if (w < g.n) {
      const float *lp0 = GSM(w) + P2_B, *num = GSM(w) + P2_MISC + PM_NUM;
      float *lp = GSM(w) + P2_LP;
      const float n0 = num[0], n1 = num[1], n2 = num[2], n3 = num[3], n4 = num[4];
      for (int i = ln; i < LP_SIZE; i += 32) {
        float sum = lp0[i];
        sum = sum + n0 * (i >= 1 ? lp0[i - 1] : 0.f);
        sum = sum + n1 * (i >= 2 ? lp0[i - 2] : 0.f);
        sum = sum + n2 * (i >= 3 ? lp0[i - 3] : 0.f);
        sum = sum + n3 * (i >= 4 ? lp0[i - 4] : 0.f);
        sum = sum + n4 * (i >= 5 ? lp0[i - 5] : 0.f);
        lp[i] = sum;
      }
    }
  GPHASE_END
  // -- P5: second 2x decimation (pitch.c:305-308) into the dead lp0 region
  GPHASE_BEGIN
    if (w < g.n) {
      const float *lp = GSM(w) + P2_LP;
      float *x4 = GSM(w) + P2_X4, *y4 = GSM(w) + P2_Y4;
      for (int j = ln; j < 240; j += 32) x4[j] = lp[384 + 2 * j];
      for (int j = ln; j < 388; j += 32) y4[j] = j < 387 ? lp[2 * j] : 0.f;
    }
  GPHASE_END
  // -- P6: coarse search, 147 lags x 240 (rnn_pitch_xcorr pitch.c:216; each lag summed in order) on 30 lanes x
  //    5 lags of the home warp with a sliding register window.  The three chain warps meanwhile run, lane =
  //    stream: find_best_pitch's running energy at quarter rate and at half rate (pitch.c:67-68, 99-100) and
  //    rnn_remove_doubling's yy_lookup (pitch.c:449-456; its prefix is xx, pitch.c:449).
  GPHASE_BEGIN
    if (w < PG) {
      if (w < g.n && ln < 30) {
        const float *x4 = GSM(w) + P2_X4, *y4 = GSM(w) + P2_Y4;
        float *xc = GSM(w) + P2_XC4;
        const float *yb = y4 + 5 * ln;
        float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        float win[5];
#pragma unroll
        for (int c = 0; c < 5; c++) win[c] = yb[c];
        for (int j0 = 0; j0 < 240; j0 += 5) {
#pragma unroll
          for (int r = 0; r < 5; r++) {
            const float xv = x4[j0 + r];
#pragma unroll
            for (int c = 0; c < 5; c++) acc[c] = acc[c] + xv * win[(c + r) % 5];
            const int nx = 5 * ln + j0 + r + 5;
            win[r] = nx < 388 ? y4[nx] : 0.f;
          }
        }
#pragma unroll
        for (int c = 0; c < 5; c++) if (5 * ln + c < 147) xc[5 * ln + c] = acc[c];
      }
    } else if (ln < g.n) {
      // Each chain consumes its inputs in register blocks of CB: the loads of a block are issued together (and,
      // in program order, before the previous block's stores, which the compiler must assume to alias), so the
      // shared-memory latency is paid once per block instead of once per step.
      float *sq = GSM(ln);
      const float *lp = sq + P2_LP;
      constexpr int CB = 7;
      if (w == PG) {                         // quarter rate: y4[j] = lp[2j]; 147 = 21 * 7 lags
        float S = 1.f;
#pragma unroll 8
        for (int j = 0; j < 240; j++) { const float v = lp[2 * j]; S = S + v * v; }
        float hi[CB], lo[CB], o[CB];
#pragma unroll
        for (int t = 0; t < CB; t++) { hi[t] = lp[2 * (t + 240)]; lo[t] = lp[2 * t]; }
        for (int i0 = 0; i0 < 147; i0 += CB) {
#pragma unroll
          for (int t = 0; t < CB; t++) { o[t] = S; S = S + (hi[t] * hi[t] - lo[t] * lo[t]); S = RMAX(1, S); }
          if (i0 + CB < 147) {
#pragma unroll
            for (int t = 0; t < CB; t++) { hi[t] = lp[2 * (i0 + CB + t + 240)]; lo[t] = lp[2 * (i0 + CB + t)]; }
          }
#pragma unroll
          for (int t = 0; t < CB; t++) sq[P2_SYY4 + i0 + t] = o[t];
        }
      } else if (w == PG + 1) {              // half rate; 294 = 42 * 7 lags
        float S = 1.f;
#pragma unroll 8
        for (int j = 0; j < 480; j++) { const float v = lp[j]; S = S + v * v; }
        float hi[CB], lo[CB], o[CB];
#pragma unroll
        for (int t = 0; t < CB; t++) { hi[t] = lp[t + 480]; lo[t] = lp[t]; }
        for (int i0 = 0; i0 < 294; i0 += CB) {
#pragma unroll
          for (int t = 0; t < CB; t++) { o[t] = S; S = S + (hi[t] * hi[t] - lo[t] * lo[t]); S = RMAX(1, S); }
          if (i0 + CB < 294) {
#pragma unroll
            for (int t = 0; t < CB; t++) { hi[t] = lp[i0 + CB + t + 480]; lo[t] = lp[i0 + CB + t]; }
          }
#pragma unroll
          for (int t = 0; t < CB; t++) sq[P2_SYY2 + i0 + t] = o[t];
        }
      } else {                               // yy_lookup; yyl[0] = xx; 384 = 48 * 8 lags
        const int N = PITCH_FRAME_SIZE / 2;
        const float *x = lp + PITCH_MAX_PERIOD / 2;
        float yy = 0.f;
#pragma unroll 8
        for (int j = 0; j < N; j++) { const float v = x[j]; yy = yy + v * v; }
        sq[P2_YYL] = yy;
        sq[P2_DOT + 0] = yy;                 // xx: the same products added in the same order (pitch.c:449-451)
        constexpr int YB = 8;
        float u[YB], v[YB], o[YB];
#pragma unroll
        for (int t = 0; t < YB; t++) { u[t] = x[-(1 + t)]; v[t] = x[N - (1 + t)]; }
        for (int i0 = 1; i0 <= PITCH_MAX_PERIOD / 2; i0 += YB) {
#pragma unroll
          for (int t = 0; t < YB; t++) { yy = yy + u[t] * u[t] - v[t] * v[t]; o[t] = RMAX(0, yy); }
          if (i0 + YB <= PITCH_MAX_PERIOD / 2) {
#pragma unroll
            for (int t = 0; t < YB; t++) { u[t] = x[-(i0 + YB + t)]; v[t] = x[N - (i0 + YB + t)]; }
          }
#pragma unroll
          for (int t = 0; t < YB; t++) sq[P2_YYL + i0 + t] = o[t];
        }
      }
    }
  GPHASE_END
  // -- P7: find_best_pitch's selection scan over the coarse lags (pitch.c:61-101), lane = stream; the home
  //    warps clear the fine-stage correlations (pitch.c:347) in the now dead x4/y4 region
  GPHASE_BEGIN
    if (w < g.n)
      for (int i = ln; i < 296; i += 32) GSM(w)[P2_XC2 + i] = 0.f;
    if (tid < g.n) {
      float *sq = GSM(tid);
      int *mi = (int *)(sq + P2_MISC + PM_INT);
      Best2 b2; best2_init(b2);
      for (int i0 = 0; i0 < 147; i0 += 7) {   // 147 = 21 * 7: inputs of a block loaded together, then visited in order
        float xc[7], sy[7];
#pragma unroll
        for (int t = 0; t < 7; t++) { xc[t] = sq[P2_XC4 + i0 + t]; sy[t] = sq[P2_SYY4 + i0 + t]; }
#pragma unroll
        for (int t = 0; t < 7; t++) best2_visit_sel(b2, i0 + t, xc[t], sy[t]);
      }
      mi[0] = b2.p0; mi[1] = b2.p1;
    }
  GPHASE_END
  // -- P8: fine search around the two coarse winners (pitch.c:344-361): 10 lags per stream, stream-minor
  GPHASE_BEGIN
    if (tid < 10 * PG && tid % PG < g.n) {
      const int q = tid % PG, c = tid / PG;
      float *sq = GSM(q);
      const int *mi = (const int *)(sq + P2_MISC + PM_INT);
      const int c0 = 2 * mi[0], c1 = 2 * mi[1];
      const int i = c < 5 ? c0 - 2 + c : c1 - 2 + (c - 5);
      bool ok = i >= 0 && i < 294;
      if (c >= 5) { int d = i - c0; if (d < 0) d = -d; if (d <= 2) ok = false; }
      if (ok) {
        const float sum = dot_seq(sq + P2_LP + 384, sq + P2_LP + i, 480);
        sq[P2_XC2 + i] = RMAX(-1, sum);
      }
    }
  GPHASE_END
  // -- P9: pick the winner, pseudo-interpolate (pitch.c:362-384), enter the half-rate domain.  Only lags with
  //    xcorr > 0 can change find_best_pitch's state, and only the <= 10 searched lags are non-zero: visit those
  //    in ascending order.
  GPHASE_BEGIN
    if (tid < g.n) {
      float *sq = GSM(tid);
      const float *xc = sq + P2_XC2, *syy = sq + P2_SYY2;
      int *mi = (int *)(sq + P2_MISC + PM_INT);
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
      mi[2] = T0;
    }
  GPHASE_END
  // -- P10: the dot products rnn_remove_doubling's candidate loop can need (pitch.c:449, 482), one lane each on
  //    the home warp: lane 1 = xy(T0), lanes 2..29 = xy(T1), xy(T1b) for k = 2..15 (xx came from the chain warp)
  GPHASE_BEGIN
    if (w < g.n && ln >= 1 && ln < 30) {
      float *sq = GSM(w);
      const float *x = sq + P2_LP + PITCH_MAX_PERIOD / 2;
      const int T0 = ((const int *)(sq + P2_MISC + PM_INT))[2];
      int off = T0, ok = 1;
      if (ln >= 2) {
        int k = 2 + (ln - 2) / 2, T1, T1b;
        rd_candidate(k, T0, &T1, &T1b);
        ok = T1 >= PITCH_MIN_PERIOD / 2;
        off = ((ln - 2) & 1) ? T1b : T1;
      }
      if (ok) sq[P2_DOT + ln] = dot_seq(x, x - off, PITCH_FRAME_SIZE / 2);
    }
  GPHASE_END
  // -- P11a: every candidate's pitch gain (pitch.c:458, 483-485: a double-precision sqrt and division each) is
  //    independent of the others: one lane per (stream, k), k = 1 (the initial candidate T0) .. 15
  GPHASE_BEGIN
    if (tid < 15 * PG && tid % PG < g.n) {
      const int q = tid % PG, k = 1 + tid / PG;
      float *sq = GSM(q);
      const float *dot = sq + P2_DOT, *yyl = sq + P2_YYL;
      const int T0 = ((const int *)(sq + P2_MISC + PM_INT))[2];
      int T1, T1b;
      rd_candidate(k, T0, &T1, &T1b);
      if (k == 1 || T1 >= PITCH_MIN_PERIOD / 2) {
        const float xy = k == 1 ? dot[1] : .5f * (dot[2 + 2 * (k - 2)] + dot[3 + 2 * (k - 2)]);
        const float yy = k == 1 ? yyl[T0] : .5f * (yyl[T1] + yyl[T1b]);
        sq[P2_CAND + k] = pitch_gain(xy, dot[0], yy);
        sq[P2_CAND + 16 + k] = xy;
        sq[P2_CAND + 32 + k] = yy;
      }
    }
  GPHASE_END
  // -- P11b: decision logic of rnn_remove_doubling (pitch.c:457-510) over the precomputed gains, lane = stream.  An
  //    accepted candidate only overwrites the running best and no threshold depends on an earlier acceptance, so
  //    walking k upwards with the gains at hand is the reference's loop.
  GPHASE_BEGIN
    if (tid < g.n) {
      float *sq = GSM(tid);
      const float *cg = sq + P2_CAND, *cxy = sq + P2_CAND + 16, *cyy = sq + P2_CAND + 32;
      int *mi = (int *)(sq + P2_MISC + PM_INT);
      const float *ps = g.pitch_state + 2 * (size_t)tid;
      const int T0 = mi[2], minperiod = PITCH_MIN_PERIOD / 2;
      const int prev_period = ((const int *)ps)[0] / 2;
      const float prev_gain = ps[1];
      float best_xy = cxy[1], best_yy = cyy[1];
      const float g0 = cg[1];
      float gg = g0;
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
        if (g1 > thresh) { best_xy = cxy[k]; best_yy = cyy[k]; Tb = T1; gg = g1; kbest = k; }
      }
      best_xy = RMAX(0, best_xy);
      float pg;
      if (best_yy <= best_xy) pg = 1.f;
      else pg = best_xy / (best_yy + 1);
      if (pg > gg) pg = gg;
      mi[3] = Tb; mi[4] = kbest;
      sq[P2_MISC + PM_F] = pg;
    }
  GPHASE_END
  // -- P12: the two refinement correlations around the chosen period (pitch.c:513-514: xcorr[k] = <x, x-(T+k-1)>,
  //    k = 0 and 2; the centre lag k = 1 was summed in P10 in the same order)
  GPHASE_BEGIN
    if (tid < 2 * PG && tid % PG < g.n) {
      const int q = tid % PG, side = tid / PG;
      float *sq = GSM(q);
      const float *x = sq + P2_LP + PITCH_MAX_PERIOD / 2;
      const int Tb = ((const int *)(sq + P2_MISC + PM_INT))[3];
      const int off = side ? Tb + 1 : Tb - 1;
      sq[P2_DOT + 32 + side] = dot_seq(x, x - off, PITCH_FRAME_SIZE / 2);
    }
  GPHASE_END
  // -- P13: final offset (pitch.c:515-524) + state update (denoise.c:369-370)
  GPHASE_BEGIN
    if (tid < g.n) {
      float *sq = GSM(tid);
      const float *dot = sq + P2_DOT;
      const int *mi = (const int *)(sq + P2_MISC + PM_INT);
      const int Tb = mi[3], kbest = mi[4];
      const float xc0 = dot[32], xc2 = dot[33];
      const float xc1 = kbest == 1 ? dot[1] : dot[2 + 2 * (kbest - 2)];
      int offset;
      if ((xc2 - xc0) > .7f * (xc1 - xc0)) offset = 1;
      else if ((xc0 - xc2) > .7f * (xc1 - xc2)) offset = -1;
      else offset = 0;
      int Tout = 2 * Tb + offset;
      if (Tout < PITCH_MIN_PERIOD) Tout = PITCH_MIN_PERIOD;
      float *ps = g.pitch_state + 2 * (size_t)tid;
      ((int *)ps)[0] = Tout;
      ps[1] = sq[P2_MISC + PM_F];
    }
  GPHASE_END
}
