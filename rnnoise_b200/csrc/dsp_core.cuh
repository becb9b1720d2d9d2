// dsp_core.cuh -- per-stream DSP stages of rnnoise_process_frame() for the GPU engine.
//
// One CTA of DSP_THREADS threads owns one stream for one frame; every stage below is written as
// a barrier-separated PHASE so that (a) on the GPU the 4 warps cooperate through shared memory and
// (b) the very same source can be executed thread-by-thread on the host by tests/emu (PHASE loops
// over tid) to check indexing and arithmetic without a GPU.  It is NOT a CPU fallback: nothing in
// the library's API reaches the host instantiation.
//
// Arithmetic contract: every float operation of the reference's scalar SSE2 DSP code
// (src/denoise.c, src/pitch.c, src/celt_lpc.c, src/kiss_fft.c) is performed in the same order
// with the same rounding -- the translation unit is compiled with --fmad=false and no fast-math,
// so X, P, band energies, pitch period and the 65 features are bit-identical to the reference.
// Parallelism comes only from operations the reference leaves independent: butterflies of one FFT
// stage, different lags of a correlation, different bands.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define HD __host__ __device__ __forceinline__
#else
#define HD static inline
#endif

// 4-byte asynchronous global -> shared copy (LDGSTS): lets a phase start fetching the data of a later
// phase without holding registers; async_wait_all() before the barrier that publishes it.  On the host
// (emulation) the copy is immediate.
HD void async_copy4(float *dst_shared, const float *src_global) {
#if defined(__CUDA_ARCH__)
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst_shared)), "l"(src_global) : "memory");
#else
  __builtin_memcpy(dst_shared, src_global, 4);   // raw bytes (the band-edge table travels through this as shorts)
#endif
}
HD void async_copy8(void *dst_shared, const void *src_global) {   // both 8-byte aligned
#if defined(__CUDA_ARCH__)
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst_shared)), "l"(src_global) : "memory");
#else
  ((float *)dst_shared)[0] = ((const float *)src_global)[0];
  ((float *)dst_shared)[1] = ((const float *)src_global)[1];
#endif
}
// 16-byte variant (both addresses 16-byte aligned): a quarter of the instructions, and .cg keeps the streamed data out
// of the small L1 these kernels leave beside their shared memory (the 4- and 8-byte forms only exist as .ca).
HD void async_copy16(float *dst_shared, const float *src_global) {
#if defined(__CUDA_ARCH__)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst_shared)), "l"(src_global) : "memory");
#else
  dst_shared[0] = src_global[0]; dst_shared[1] = src_global[1]; dst_shared[2] = src_global[2]; dst_shared[3] = src_global[3];
#endif
}
// Streaming loads / stores for the bulk per-stream arrays (spectra, ring, overlap memory, PCM): evict-first, so that
// they do not push the few KB of shared tables (twiddles, window, band weights, DCT) out of the small L1 these kernels
// leave beside their shared memory.  Plain accesses in the host emulation.
HD float ld_stream(const float *p) {
#if defined(__CUDA_ARCH__)
  return __ldcs(p);
#else
  return *p;
#endif
}
// plain global load that bypasses L1 (the history ring: read here once, re-read from L2 by the next kernel).  Like
// ld_stream it names the global space, which lets the compiler move it above shared-memory stores.
HD float ld_global(const float *p) {
#if defined(__CUDA_ARCH__)
  return __ldcg(p);
#else
  return *p;
#endif
}
HD void st_stream(float *p, float v) {
#if defined(__CUDA_ARCH__)
  __stcs(p, v);
#else
  *p = v;
#endif
}
HD void st_stream2(float *p, float a, float b) {   // p 8-byte aligned
#if defined(__CUDA_ARCH__)
  __stcs((float2 *)p, make_float2(a, b));
#else
  p[0] = a; p[1] = b;
#endif
}
HD void async_wait_all() {
#if defined(__CUDA_ARCH__)
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
#endif
}

#define DSP_THREADS 128
#define FRAME_SIZE 480
#define WINDOW_SIZE 960
#define FREQ_SIZE 481
#define NB_BANDS 32
#define NB_FEATURES 65
#define TRAIN_RECORD (NB_FEATURES + NB_BANDS + 1)   // features | ideal gains | vad target (dump_features.c:487-489)
#define PITCH_MIN_PERIOD 60
#define PITCH_MAX_PERIOD 768
#define PITCH_FRAME_SIZE 960
#define PITCH_BUF_SIZE 1728
#define LP_SIZE 864

// Same operand orientation as the reference's MAX16/MIN16/MAX32 macros (src/arch.h:72-75).
#define RMAX(a, b) ((a) > (b) ? (a) : (b))
#define RMIN(a, b) ((a) < (b) ? (a) : (b))

struct cpx { float r, i; };

// Tables, generated on the host from the reference's closed forms (dsp_tables.c) and kept in
// global memory (lane-divergent indices would serialise in __constant__).
struct DspTables {
  float half_window[FRAME_SIZE];   // src/dump_rnnoise_tables.c:85
  float dct[NB_BANDS * NB_BANDS];  // :92-97
  cpx tw[WINDOW_SIZE];             // src/kiss_fft.c:406-420
  short bitrev[WINDOW_SIZE];       // digit reversal for radices 5,3,4,4,4
  short eband[NB_BANDS + 2];       // src/denoise.c:63-65
  unsigned char bin_band[400];     // triangular segment (0..32) that holds bin k
  float bin_frac[400];             // (float)j / band_size of bin k inside its segment (denoise.c:100,148)
  float bin_cfrac[400];            // 1 - bin_frac[k], the weight towards the lower band (denoise.c:103)
  float fft_scale;                 // rnnoise_tables.c:562 literal
};

// ------------------------------------------------------------------------------------------------
// Shared-memory plans (floats).  The analysis of one frame is two kernels, each CTA = one stream:
//   pitch kernel    : whitened half-rate signal + search scratch          (SM_PITCH_END + SM_MISC_SIZE)
//   spectrum kernel : FFT work buffer + a copy of X for the X.P correlation (SM_SPEC_END + SM_MISC_SIZE)
// The pitch history itself stays in HBM/L2 (ring): the pitch kernel stages it once (aligned 16-byte asynchronous
// copies, logical order) for the decimation, the spectrum kernel fetches its two analysis windows the same way.
// ------------------------------------------------------------------------------------------------
//   pitch kernel
#define SM_LP 0                          // [864] whitened half-rate signal
#define SM_LP0 (SM_LP + LP_SIZE)         // [864] second half of the raw-history staging [SM_LP, SM_LP + 1728) of the first phase (the decimated
                                         //       signal before whitening is SM_LP0N); x4 / y4 / xcorr ... overlay it afterwards
#define SM_X4 (SM_LP0)                   // [240]   (reuses LP0 once the FIR is done)
#define SM_Y4 (SM_X4 + 240)              // [388]
#define SM_XC (SM_Y4 + 388)              // [296] coarse / fine correlations
#define SM_SYY (SM_XC + 296)             // [296] running energies seen by find_best_pitch
#define SM_YYL (SM_SYY + 296)            // [392] yy_lookup
#define SM_DOT (SM_YYL + 392)            // [64]  remove_doubling dot products
#define SM_PITCH_END (SM_DOT + 64)
#define SM_LP0N (SM_LP0 + LP_SIZE)       // [864] k_pitch: the decimated signal before whitening lives behind the raw history that
                                         //       lp | lp0 stage at first -- over the (then idle) tail of the search scratch and
                                         //       the first 52 floats of the misc block, whose slots (MI_*) start at 64
//   spectrum kernel
#define SM_F 0                           // [1920] FFT work buffer (interleaved complex)
#define SM_XS (SM_F + 2 * WINDOW_SIZE)   // [800] bins 0..399 of X kept for the X.P correlation (the band sums end at bin 400)
#define SM_WIN (SM_XS + 2 * 400)         // [964] analysis window staged from the ring in 16-byte pieces (the pitch-lagged one starts
                                         //       0..3 floats into the first piece); after the P transform: the weighted per-bin terms
                                         //       of Re(X conj P), interleaved (frac, 1 - frac) pairs [0,800)
#define SM_SPEC_END (SM_WIN + WINDOW_SIZE + 4)
#define SM_MISC_SIZE 288                 // pitch kernel: small per-stream scalars / vectors after its plan (MI_*)
#define SM_SPEC_MISC 228                 // spectrum kernel: its own, tighter misc block (SMI_*)
#define SM_PITCH_TOTAL (SM_PITCH_END + SM_MISC_SIZE)
#define SM_SPEC_TOTAL (SM_SPEC_END + SM_SPEC_MISC)   // 3912 floats = 15.3 KB (registers, not shared memory, set the CTAs per SM: engine.cu)
// misc slots (float indices relative to the misc base)
#define MI_AC 64    // [5] autocorrelation
#define MI_NUM 72   // [5] whitening FIR taps
#define MI_INT 80   // ints: [0]=best0 [1]=best1 [2]=T (pitch index) [3]=silence [4]=T0 half-rate [5]=Tb [6]=kbest
// spectrum kernel's misc block
#define SMI_INT 0    // ints: [3]=silence
#define SMI_BAND 8   // [3][34] band sums (X, P, X.P)
#define SMI_LY 8     // [32] log band energies -- written after the band sums are consumed, in their place
#define SMI_E 112    // [3][32] Ex, Ep, Exp
#define SMI_EBAND 208 // [34] shorts: band edges staged from the table (the band-sum lanes' loop bounds)
static_assert(SM_WIN % 4 == 0 && SM_XS % 4 == 0 && SM_SPEC_END % 4 == 0 && SMI_LY % 4 == 0 && SMI_E % 4 == 0, "16-byte pieces / vector loads");
static_assert(SM_LP0 + LP_SIZE <= SM_PITCH_END, "lp0 overlay");
static_assert(SM_LP0N % 4 == 0 && SM_LP0N + LP_SIZE <= SM_PITCH_END + 64, "k_pitch: decimated signal ends before the misc slots");
static_assert(SM_LP % 4 == 0 && SM_X4 % 4 == 0 && SM_Y4 % 4 == 0 && SM_SYY % 4 == 0 && (SM_LP + 384) % 4 == 0,
              "single-lane chains use 16-byte vector loads");

// logical sample k of the updated 1728-sample pitch history (after this frame's shift)
HD int ring_pos(int ring_base, int k) {
  int p = ring_base + k;
  if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
  return p;
}
HD float ring_at(const float *ring, int ring_base, int k) {
  int p = ring_base + k;
  if (p >= PITCH_BUF_SIZE) p -= PITCH_BUF_SIZE;
  return ring[p];
}

// ------------------------------------------------------------------------------------------------
// 960-point forward FFT stages (src/kiss_fft.c:101-316; stage order rnn_fft_impl:518-564).
// ------------------------------------------------------------------------------------------------
HD cpx cmul(cpx a, cpx b) {
  cpx m;
  m.r = a.r * b.r - a.i * b.i;
  m.i = a.r * b.i + a.i * b.r;
  return m;
}
HD cpx cadd(cpx a, cpx b) { cpx m; m.r = a.r + b.r; m.i = a.i + b.i; return m; }
HD cpx csub(cpx a, cpx b) { cpx m; m.r = a.r - b.r; m.i = a.i - b.i; return m; }

// The work buffer F is addressed through an XOR swizzle inside its 16-element blocks: element idx lives at
//   fsw(idx) = idx ^ (((idx >> 4) & 3) << 2),
// a permutation of each aligned block of 16 that moves the four 4-element groups of block B by B mod 4 places.  The
// second stage (radix 4, m = 4) reads elements 16 g + j + 4 q with (g, j) = lane: unswizzled, the 16 lanes of a half
// warp hit only 4 of the 16 8-byte bank pairs (a 4-way conflict on all 8 accesses of a butterfly: 3x the wavefronts
// of that stage, a quarter of all shared-memory wavefronts of the spectrum and synthesis kernels);
// swizzled, bank = j + 4 (q ^ (g & 3)) takes all 16 values.  The other stages walk j or u linearly inside a block
// (the XOR is then a constant per half warp) and stay conflict-free; stage 1 still writes 4 contiguous elements.
// Arithmetic and results are untouched: only where an element is parked between stages changes.
HD int fsw(int idx) { return idx ^ (((idx >> 4) & 3) << 2); }

// Stage 1 (radix 4, m = 1) fused with the bit-reversed, scaled, windowed load: group g gathers
// its four inputs straight from `src` (kiss_fft.c:577-584 + kf_bfly4 m==1 branch :112-130).
// Input element i of the transform is win(i) * src[i] (imag 0) when `herm` is null, or the
// Hermitian extension of herm[0..480] (inverse_transform, denoise.c:200-211).
// `hw` = the half window (the table itself, or a copy a kernel staged into shared memory).
HD void fft_stage1(cpx *F, const float *src, const cpx *herm, const DspTables *T, int tid, int nthr, const float *hw = nullptr) {
  if (!hw) hw = T->half_window;
  for (int g = tid; g < 240; g += nthr) {
    int j0 = g / 48, j1 = (g / 16) % 3, j2 = (g / 4) % 4, j3 = g % 4;
    int base = j0 + 5 * j1 + 15 * j2 + 60 * j3;
    cpx a[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      int i = base + 240 * q;
      cpx v;
      if (herm) {
        if (i < FREQ_SIZE) v = herm[i];
        else { v.r = herm[WINDOW_SIZE - i].r; v.i = -herm[WINDOW_SIZE - i].i; }
      } else {
        int wi = i < FRAME_SIZE ? i : WINDOW_SIZE - 1 - i;
        v.r = src[i] * hw[wi];
        v.i = 0.f;
      }
      a[q].r = T->fft_scale * v.r;
      a[q].i = T->fft_scale * v.i;
    }
    cpx s0 = csub(a[0], a[2]);
    a[0] = cadd(a[0], a[2]);
    cpx s1 = cadd(a[1], a[3]);
    a[2] = csub(a[0], s1);
    a[0] = cadd(a[0], s1);
    s1 = csub(a[1], a[3]);
    a[1].r = s0.r + s1.i; a[1].i = s0.i - s1.r;
    a[3].r = s0.r - s1.i; a[3].i = s0.i + s1.r;
    cpx *Fo = F + 16 * (g >> 2) + 4 * ((g & 3) ^ ((g >> 2) & 3));   // fsw(4 g .. 4 g + 3): still 4 contiguous elements
    Fo[0] = a[0]; Fo[1] = a[1]; Fo[2] = a[2]; Fo[3] = a[3];
  }
}
// radix-4 stages 2 and 3: m = 4 (groups 16 apart, twiddle stride 60) or m = 16 (groups 64 apart, stride 15).
// Element q of butterfly (g, j) is F[g * gstride + j + q * m]; its swizzled place is
//   m = 4 : 16 g + j + 4 (q ^ (g & 3))          m = 16 : 64 g + 16 q + (j ^ 4 q)
HD void fft_radix4(cpx *F0, int m, int gstride, int fs, const DspTables *T, int tid, int nthr) {
  for (int b = tid; b < 240; b += nthr) {
    int g = b / m, j = b % m;
    cpx *F = F0 + g * gstride;
    int i0, i1, i2, i3;
    if (m == 4) {
      const int s = (g & 3) << 2;
      i0 = j + s; i1 = j + (4 ^ s); i2 = j + (8 ^ s); i3 = j + (12 ^ s);
    } else {
      i0 = j; i1 = 16 + (j ^ 4); i2 = 32 + (j ^ 8); i3 = 48 + (j ^ 12);
    }
    cpx s0 = cmul(F[i1], T->tw[j * fs]);
    cpx s1 = cmul(F[i2], T->tw[2 * j * fs]);
    cpx s2 = cmul(F[i3], T->tw[3 * j * fs]);
    cpx f0 = F[i0];
    cpx s5 = csub(f0, s1);
    f0 = cadd(f0, s1);
    cpx s3 = cadd(s0, s2);
    cpx s4 = csub(s0, s2);
    F[i2] = csub(f0, s3);
    F[i0] = cadd(f0, s3);
    cpx o1, o3;
    o1.r = s5.r + s4.i; o1.i = s5.i - s4.r;
    o3.r = s5.r - s4.i; o3.i = s5.i + s4.r;
    F[i1] = o1; F[i3] = o3;
  }
}
HD void fft_radix3(cpx *F0, const DspTables *T, int tid, int nthr) { // m = 64, 5 groups of 192
  const int m = 64, fs = 5;
  const float epi3 = T->tw[fs * m].i;
  for (int b = tid; b < 320; b += nthr) {
    int g = b / m, j = b % m;
    cpx *F = F0 + g * 192 + fsw(j);   // 192 g and 64 q leave (idx >> 4) & 3 unchanged: the swizzle is that of j
    cpx s1 = cmul(F[m], T->tw[j * fs]);
    cpx s2 = cmul(F[2 * m], T->tw[2 * j * fs]);
    cpx s3 = cadd(s1, s2);
    cpx s0 = csub(s1, s2);
    cpx f0 = F[0], f1;
    f1.r = f0.r - s3.r * .5f;
    f1.i = f0.i - s3.i * .5f;
    s0.r *= epi3; s0.i *= epi3;
    F[0] = cadd(f0, s3);
    cpx o2, o1;
    o2.r = f1.r + s0.i; o2.i = f1.i - s0.r;
    o1.r = f1.r - s0.i; o1.i = f1.i + s0.r;
    F[2 * m] = o2; F[m] = o1;
  }
}
HD void fft_radix5(cpx *F, const DspTables *T, int tid, int nthr) { // m = 192, one group
  const int m = 192;
  const cpx ya = T->tw[m], yb = T->tw[2 * m];
  for (int u = tid; u < m; u += nthr) {
    const int v = fsw(u);   // 192 q leaves (idx >> 4) & 3 unchanged
    cpx s0 = F[v];
    cpx s1 = cmul(F[v + m], T->tw[u]);
    cpx s2 = cmul(F[v + 2 * m], T->tw[2 * u]);
    cpx s3 = cmul(F[v + 3 * m], T->tw[3 * u]);
    cpx s4 = cmul(F[v + 4 * m], T->tw[4 * u]);
    cpx s7 = cadd(s1, s4), s10 = csub(s1, s4), s8 = cadd(s2, s3), s9 = csub(s2, s3);
    cpx o0;
    o0.r = s0.r + (s7.r + s8.r);
    o0.i = s0.i + (s7.i + s8.i);
    F[v] = o0;
    cpx s5, s6, s11, s12;
    s5.r = s0.r + (s7.r * ya.r + s8.r * yb.r);
    s5.i = s0.i + (s7.i * ya.r + s8.i * yb.r);
    s6.r = s10.i * ya.i + s9.i * yb.i;
    s6.i = -(s10.r * ya.i + s9.r * yb.i);
    F[v + m] = csub(s5, s6);
    F[v + 4 * m] = cadd(s5, s6);
    s11.r = s0.r + (s7.r * yb.r + s8.r * ya.r);
    s11.i = s0.i + (s7.i * yb.r + s8.i * ya.r);
    s12.r = s9.i * ya.i - s10.i * yb.i;
    s12.i = s10.r * yb.i - s9.r * ya.i;
    F[v + 2 * m] = cadd(s11, s12);
    F[v + 3 * m] = csub(s11, s12);
  }
}

// ------------------------------------------------------------------------------------------------
// Band sums (compute_band_energy / compute_band_corr, src/denoise.c:90-138).  Thread b owns
// sum[b] (b = 0..33) and adds its terms in the reference's order: first the frac*t terms of band
// b-1, then the (1-frac)*t terms of band b.  which: 0 -> |A|^2, 1 -> Re(A conj B).
// ------------------------------------------------------------------------------------------------
HD float band_sum_one(int b, const cpx *A, const cpx *B, const DspTables *T) {
  float sum = 0.f;
  if (b >= 1) {
    for (int k = T->eband[b - 1]; k < T->eband[b]; k++) {
      const float frac = T->bin_frac[k];      // == (float)j / band_size, tabulated (no divide in the loop)
      cpx a = A[k], c = B[k];
      float t = a.r * c.r;
      t += a.i * c.i;
      sum += frac * t;
    }
  }
  if (b <= NB_BANDS) {
    for (int k = T->eband[b]; k < T->eband[b + 1]; k++) {
      const float frac = T->bin_frac[k];
      cpx a = A[k], c = B[k];
      float t = a.r * c.r;
      t += a.i * c.i;
      sum += (1 - frac) * t;
    }
  }
  return sum;
}
// Same sums from per-bin terms t[k] precomputed by parallel lanes (t = a.r*c.r; t += a.i*c.i, exactly
// as above) and tabulated weights: leaves two loads + FMUL + FADD per step on the serial lanes.
HD float band_sum_terms(int b, const float *t, const DspTables *T) {
  float sum = 0.f;
  if (b >= 1)
    for (int k = T->eband[b - 1]; k < T->eband[b]; k++) sum += T->bin_frac[k] * t[k];
  if (b <= NB_BANDS)
    for (int k = T->eband[b]; k < T->eband[b + 1]; k++) sum += T->bin_cfrac[k] * t[k];
  return sum;
}
// Same sums again with the weights already applied by the parallel lanes: w[k * stride] = bin_frac[k] * t[k]
// and w[k * stride + coff] = bin_cfrac[k] * t[k] (the very products of the loop above), which leaves one
// shared-memory load + FADD per step on the serial lanes and no table load at all.
// The sums are serial float chains of up to 83 terms on one lane each: the terms are loaded eight at a time (all in
// flight together) and then added in order, so that a lane pays one shared-memory latency per eight steps instead of
// one per step.  `eb` = band edges (the table, or a staged copy).
HD float band_chain8(float sum, const float *p, int stride, int n) {
  for (; n >= 8; n -= 8, p += 8 * stride) {
    float t[8];
#pragma unroll
    for (int u = 0; u < 8; u++) t[u] = p[u * stride];
#pragma unroll
    for (int u = 0; u < 8; u++) sum += t[u];
  }
  if (n >= 4) {
    float t[4];
#pragma unroll
    for (int u = 0; u < 4; u++) t[u] = p[u * stride];
#pragma unroll
    for (int u = 0; u < 4; u++) sum += t[u];
    n -= 4; p += 4 * stride;
  }
  for (; n > 0; n--, p += stride) sum += p[0];
  return sum;
}
HD float band_sum_pre(int b, const float *w, int stride, int coff, const short *eb) {
  float sum = 0.f;
  const int k1 = eb[b];
  if (b >= 1) { const int k0 = eb[b - 1]; sum = band_chain8(sum, w + k0 * stride, stride, k1 - k0); }
  if (b <= NB_BANDS) { const int k2 = eb[b + 1]; sum = band_chain8(sum, w + k1 * stride + coff, stride, k2 - k1); }
  return sum;
}
HD float bin_term(cpx a, cpx c) {
  float t = a.r * c.r;
  t += a.i * c.i;
  return t;
}
// sum[34] -> E[32] with the edge-band fix-up (denoise.c:107-112)
HD float band_finish(const float *sum, int b) {
  if (b == 0) return (sum[0] + sum[1]) * 2 / 3;
  if (b == NB_BANDS - 1) return (sum[NB_BANDS] + sum[NB_BANDS + 1]) * 2 / 3;
  return sum[b + 1];
}

// interp_band_gain (denoise.c:140-154) evaluated per bin; bins >= 400 are 0 (callers zero-init).
HD float interp_bin(const float *band, int k, const DspTables *T) {
  if (k >= 400) return 0.f;
  if (k < 2) return band[0];
  if (k >= 356) return band[NB_BANDS - 1];
  int b = T->bin_band[k];
  float frac = T->bin_frac[k];
  return (1 - frac) * band[b - 1] + frac * band[b];
}

// dct (denoise.c:160-170): output i, sequential over j
HD float dct_one(const float *in, int i, const DspTables *T) {
  float sum = 0.f;
  for (int j = 0; j < NB_BANDS; j++) sum += in[j] * T->dct[j * NB_BANDS + i];
  return (float)(sum * sqrt(2. / 22));
}

// same with the table already staged (row-major [j][i], as T->dct)
HD float dct_one_tab(const float *in, int i, const float *tab) {
  float sum = 0.f;
#pragma unroll 8
  for (int j = 0; j < NB_BANDS; j++) sum += in[j] * tab[j * NB_BANDS + i];
  return (float)(sum * sqrt(2. / 22));
}

// one biquad step (rnn_biquad, denoise.c:409-419; b = {-2, 1}, a = {-1.99599, 0.996} :469-470)
HD float biquad_step(float xi, float &m0, float &m1) {
  const float b0 = -2.f, b1 = 1.f, a0 = -1.99599f, a1 = 0.99600f;
  float yi = xi + m0;
  m0 = (float)((double)m1 + ((double)b0 * (double)xi - (double)a0 * (double)yi));
  m1 = (float)((double)b1 * (double)xi - (double)a1 * (double)yi);
  return yi;
}

// compute_pitch_gain (src/pitch.c:416-419)
HD float pitch_gain(float xy, float xx, float yy) { return (float)(xy / sqrt((double)(1 + xx * yy))); }

// find_best_pitch's selection scan (src/pitch.c:61-101) over precomputed running energies syy[i]
// (= the value of Syy when lag i is examined).
// 16-byte vector view for single-lane chains (one LDS.128 / STS.128 per four elements)
struct alignas(16) f4 { float x, y, z, w; };

// s + x[0]*y[0] + x[1]*y[1] + ... + x[n-1]*y[n-1], added strictly in index order (the reference's summation order),
// n % 4 == 0, n >= 4.  The n dependent additions are the critical path of the narrow pitch phases and one warp does
// not hide its own shared-memory latency, so the operands travel in two register sets of four: the loads of block
// b+1 are in flight while block b is added (software pipelining by hand, unrolled twice so that no register copies
// are needed; same instruction count as the plain loop).
#define DC_LOAD(xr, yr, i0) { xr[0] = x[(i0)]; xr[1] = x[(i0) + 1]; xr[2] = x[(i0) + 2]; xr[3] = x[(i0) + 3]; \
                              yr[0] = y[(i0)]; yr[1] = y[(i0) + 1]; yr[2] = y[(i0) + 2]; yr[3] = y[(i0) + 3]; }
#define DC_ACC(xr, yr) { s = s + xr[0] * yr[0]; s = s + xr[1] * yr[1]; s = s + xr[2] * yr[2]; s = s + xr[3] * yr[3]; }
HD float dot_chain4(float s, const float *x, const float *y, int n) {
  const int B = n >> 2;
  float xa[4], ya[4], xb[4], yb[4];
  DC_LOAD(xa, ya, 0)
  int b = 0;
  for (; b + 2 < B; b += 2) {
    DC_LOAD(xb, yb, 4 * b + 4)
    DC_ACC(xa, ya)
    DC_LOAD(xa, ya, 4 * b + 8)
    DC_ACC(xb, yb)
  }
  if (B - b == 2) {
    DC_LOAD(xb, yb, 4 * b + 4)
    DC_ACC(xa, ya)
    DC_ACC(xb, yb)
  } else {
    DC_ACC(xa, ya)
  }
  return s;
}
#undef DC_LOAD
#undef DC_ACC

// Running energy chain of find_best_pitch (pitch.c:67-68, 99-100), split so that only the truly
// serial part runs on one lane:
//   prefix : S = 1 + sum_{j<len} y[j]^2, added in index order (len % 4 == 0, y 16-byte aligned)
//   running: syy[i] = S_i,  S_{i+1} = max(1, S_i + d[i]) with d[i] = y[i+len]^2 - y[i]^2 precomputed
//            by parallel lanes into the same array (read d[i], then overwrite it with S_i).
HD float sq_prefix(float S, const float *y, int len) {
  for (int j = 0; j < len; j += 4) {
    f4 v = *(const f4 *)(y + j);
    S = S + v.x * v.x; S = S + v.y * v.y; S = S + v.z * v.z; S = S + v.w * v.w;
  }
  return S;
}
HD void syy_running_inplace(float *syy_d, float S, int max_pitch) {
  int i = 0;
  for (; i + 4 <= max_pitch; i += 4) {
    f4 d = *(const f4 *)(syy_d + i), o;
    o.x = S; S = S + d.x; S = RMAX(1, S);
    o.y = S; S = S + d.y; S = RMAX(1, S);
    o.z = S; S = S + d.z; S = RMAX(1, S);
    o.w = S; S = S + d.w; S = RMAX(1, S);
    *(f4 *)(syy_d + i) = o;
  }
  for (; i < max_pitch; i++) {
    float d = syy_d[i];
    syy_d[i] = S;
    S = S + d; S = RMAX(1, S);
  }
}
// find_best_pitch's update for one examined lag (pitch.c:71-98)
struct Best2 { float num0, num1, den0, den1; int p0, p1; };
HD void best2_init(Best2 &b) { b.num0 = -1; b.num1 = -1; b.den0 = 0; b.den1 = 0; b.p0 = 0; b.p1 = 1; }
HD void best2_visit(Best2 &b, int i, float xcorr, float Syy) {
  if (xcorr > 0) {
    float x16 = xcorr;
    x16 *= 1e-12f;
    float num = x16 * x16;
    if (num * b.den1 > b.num1 * Syy) {
      if (num * b.den0 > b.num0 * Syy) {
        b.num1 = b.num0; b.den1 = b.den0; b.p1 = b.p0;
        b.num0 = num; b.den0 = Syy; b.p0 = i;
      } else {
        b.num1 = num; b.den1 = Syy; b.p1 = i;
      }
    }
  }
}

// find_best_pitch's update for one examined lag (pitch.c:71-98; best2_visit of dsp_core.cuh) without branches: lanes of
// a warp hold different streams here, and three nested divergent branches per lag cost ~200 cycles per step.  The
// products are formed unconditionally (no side effects) and the reference's conditions select the updates.
HD void best2_visit_sel(Best2 &b, int i, float xcorr, float Syy) {
  float x16 = xcorr;
  x16 *= 1e-12f;
  const float num = x16 * x16;
  const bool c1 = xcorr > 0 && (num * b.den1 > b.num1 * Syy);
  const bool c0 = c1 && (num * b.den0 > b.num0 * Syy);
  b.num1 = c0 ? b.num0 : c1 ? num : b.num1;
  b.den1 = c0 ? b.den0 : c1 ? Syy : b.den1;
  b.p1 = c0 ? b.p0 : c1 ? i : b.p1;
  b.num0 = c0 ? num : b.num0;
  b.den0 = c0 ? Syy : b.den0;
  b.p0 = c0 ? i : b.p0;
}

// Order-4 whitening filter design (src/pitch.c:181-212, src/celt_lpc.c:38-89): ac[5] -> taps[5]
HD void lpc_taps(const float *ac_in, float *num) {
  float ac[5];
  for (int k = 0; k < 5; k++) ac[k] = ac_in[k];
  ac[0] *= 1.0001f;
  for (int i = 1; i <= 4; i++) ac[i] -= ac[i] * (.008f * i) * (.008f * i);
  float lpc[4] = {0, 0, 0, 0};
  float error = ac[0];
  if (ac[0] != 0) {
    for (int i = 0; i < 4; i++) {
      float rr = 0;
      for (int j = 0; j < i; j++) rr += lpc[j] * ac[i - j];
      rr += ac[i + 1];
      float r = -rr / error;
      lpc[i] = r;
      for (int j = 0; j < (i + 1) >> 1; j++) {
        float t1 = lpc[j], t2 = lpc[i - 1 - j];
        lpc[j] = t1 + r * t2;
        lpc[i - 1 - j] = t2 + r * t1;
      }
      error = error - (r * r) * error;
      if (error < .001f * ac[0]) break;
    }
  }
  float tmp = 1.f;
  for (int i = 0; i < 4; i++) {
    tmp = .9f * tmp;
    lpc[i] = lpc[i] * tmp;
  }
  const float c1 = .8f;
  num[0] = lpc[0] + .8f;
  num[1] = lpc[1] + c1 * lpc[0];
  num[2] = lpc[2] + c1 * lpc[1];
  num[3] = lpc[3] + c1 * lpc[2];
  num[4] = c1 * lpc[3];
}

// Candidate geometry of rnn_remove_doubling (src/pitch.c:462-481), half-rate domain.
// k = 1 stands for the initial candidate T0 itself.
HD void rd_candidate(int k, int T0, int *T1, int *T1b) {
  const int maxperiod = PITCH_MAX_PERIOD / 2;
  if (k == 1) { *T1 = T0; *T1b = T0; return; }
  // second_check[k] of pitch.c:420 for 2 <= k <= 15 = {3,2,3,2,5,2,3,2,3,2,3,2,5,2}: computed, so that no
  // per-lane indexed table ends up in local memory
  const int sc = (k & 1) ? 2 : (k == 6 || k == 12) ? 5 : 3;
  // n / (2k), 0 <= n < 4096, 4 <= 2k <= 30, without a hardware integer division by a per-lane divisor:
  // trunc((n + 0.5) * (1 / 2k)) in float.  The fractional part of (n + 0.5) / 2k lies in [1/60, 59/60], far
  // beyond the rounding error (< 2^-11) of the two float operations, so the truncation is exact
  // (checked exhaustively over the whole domain in tests/test_dsp_emulation.py).
#ifdef RD_INT_DIV
  int t1 = (2 * T0 + k) / (2 * k);
  *T1 = t1;
  if (k == 2) *T1b = (t1 + T0 > maxperiod) ? T0 : T0 + t1;
  else *T1b = (2 * sc * T0 + k) / (2 * k);
#else
  const float inv = 1.0f / (float)(2 * k);
  int t1 = (int)(((float)(2 * T0 + k) + 0.5f) * inv);
  *T1 = t1;
  if (k == 2) *T1b = (t1 + T0 > maxperiod) ? T0 : T0 + t1;
  else *T1b = (int)(((float)(2 * sc * T0 + k) + 0.5f) * inv);
#endif
}
