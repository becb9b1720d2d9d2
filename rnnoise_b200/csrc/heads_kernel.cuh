// heads_kernel.cuh -- output heads of the network, register-tiled (default kernel; k_heads in
// rnn_kernels.cuh is the cp.async cross-check with the same arithmetic).
//
//   cat = [conv2_out | gru1 | gru2 | gru3]  (rnn.c:53-57), K = 4 * gru inputs
//   gains[32] = sigmoid(dense_out . cat + b)   each output one sequential FMA chain over K (sgemv, vec_avx.h:672)
//   vad       = sigmoid(vad_dense . cat + b)   scalar loop: multiply, then add (vec_avx.h:731-735)
//
// CTA = 2 * NS * NW streams, NW compute warps + 1.  Compute warp w owns 2 * NS streams x 32 outputs: a thread keeps NS
// streams x 2 adjacent outputs = 2 * NS independent chains in registers, so one LDS.128 of activations and one LDS.64
// of weights feed 8 / NS FMAs.  The kernel is bound by the latency of its serial FMA chains, not by loads: with one
// compute warp per scheduler (NW = 4) nothing hides a warp's shared-memory and dependent-issue stalls, so the
// 32-stream tile comes in two shapes -- <4, 4> (8 chains per thread) and <2, 8> (4 chains per thread, two warps per
// scheduler: same streams per CTA, same number of SMs taken, half the work per warp).  <2, 4> (16 streams per CTA)
// launches twice the CTAs.  The last warp runs the VAD chains (lane = stream) and is the producer: inputs and
// weights arrive in chunks of 64 inputs (16-byte cp.async pieces of the weight slab and of the activation rows, all
// completing on one mbarrier) through an H2_STAGES-deep ring, so staging costs no instructions on the compute warps.
// grid = ceil(S / TS); dynamic smem = H2_STAGES * (TS * 272 + 8192) B + 16 KB.
#pragma once
#include "gru_tc.cuh"

#define H2_TS 32
#define H2_KC 64
#define H2_XS (H2_KC + 4)   // padded row: 272 B keeps rows 16-byte aligned and LDS.128 conflict-free
#ifndef H2_STAGES
#define H2_STAGES 6
#endif
template <int TS> struct H2StageT {
  float xs[TS][H2_XS];
  float ws[H2_KC][NB_GAINS];
};
#define H2_MAX_K 4096   // 4 * gru, gru <= 1024: the VAD weight vector is staged whole, once
template <int NS, int NW = 4> constexpr int h2_smem_bytes() { return H2_STAGES * (int)sizeof(H2StageT<2 * NS * NW>) + H2_MAX_K * 4 + 128; }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <int NS, int NW>
__global__ void __launch_bounds__(32 * NW + 32) k_heads2(int S, DevModel m, const float *__restrict__ c2,
                                                const float *__restrict__ g1, const float *__restrict__ g2,
                                                const float *__restrict__ g3, const int *__restrict__ silence,
                                                float *__restrict__ gains, float *__restrict__ vad,
                                                float *__restrict__ vad_user, int vad_stride) {
  extern __shared__ __align__(128) uint8_t h2_smem[];
  constexpr int TS = 2 * NS * NW, NT = 32 * NW + 32;
  typedef H2StageT<TS> H2Stage;
  H2Stage *st = (H2Stage *)h2_smem;
  float *wv_all = (float *)(h2_smem + H2_STAGES * sizeof(H2Stage));   // [4 * gru] vad_dense weights
  __shared__ __align__(8) uint64_t full[H2_STAGES];
  const int s0 = blockIdx.x * TS, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gru = m.gru, nchunk = 4 * gru / H2_KC;
  const int live_rows = min(TS, S - s0);
  if (tid == 0) {
    for (int i = 0; i < H2_STAGES; i++) mbar_init(smem_u32(&full[i]), 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  pdl_trigger();
  for (int i = tid; i < gru; i += NT) cp_async16(&wv_all[4 * i], m.vad_dense.w + 4 * i, true);   // 4 * gru floats
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  pdl_wait();   // GRU-3 state of this frame
  __syncthreads();
  // producer (warp NW): chunk c -> stage c % H2_STAGES.  gru % 64 == 0, so a chunk never straddles two sources.
  // Everything travels as 16-byte cp.async pieces issued by the 32 lanes (activation rows of 256 B per stream into
  // the padded rows, the 8 KB weight slab) rather than bulk copies, which have a fixed cost each on the SM's copy
  // engine whatever their size, and two of them per chunk (weights + VAD weights) would dominate the FMA chain.  Each lane's cp.async.mbarrier.arrive.noinc fires once its pieces have landed: 32 arrivals per phase.
  auto produce = [&](int c) {
    const int buf = c % H2_STAGES, c0 = c * H2_KC, src = c0 / gru, off = c0 - src * gru;
    const uint32_t bar = smem_u32(&full[buf]);
    const float *wsrc = m.dense_out.w + (size_t)c0 * NB_GAINS;
#pragma unroll
    for (int i = 0; i < H2_KC * NB_GAINS / 4 / 32; i++) {   // 512 pieces of the [64][32] weight slab, contiguous in memory
      const int piece = i * 32 + lane;
      cp_async16(&st[buf].ws[0][0] + 4 * piece, wsrc + 4 * piece, true);
    }
    const float *p = (src == 0 ? c2 : src == 1 ? g1 : src == 2 ? g2 : g3) + (size_t)s0 * gru + off;
#pragma unroll
    for (int i = 0; i < TS * H2_KC / 4 / 32; i++) {   // piece = i * 32 + lane: row = piece / 16, 16-byte column = piece % 16
      const int row = 2 * i + (lane >> 4), col = lane & 15;
      cp_async16(&st[buf].xs[row][4 * col], p + (size_t)(row < live_rows ? row : 0) * gru + 4 * col, row < live_rows);
    }
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
  };
  if (warp == NW)
    for (int c = 0; c < H2_STAGES - 1 && c < nchunk; c++) produce(c);
  float acc[NS][2];
#pragma unroll
  for (int i = 0; i < NS; i++) acc[i][0] = acc[i][1] = 0.f;
  float y = 0.f;
  const int row0 = warp * (2 * NS) + (lane >> 4) * NS, o2 = (lane & 15) * 2;
  for (int c = 0; c < nchunk; c++) {
    const int buf = c % H2_STAGES;
    if (warp == NW && c + H2_STAGES - 1 < nchunk) produce(c + H2_STAGES - 1);   // that stage was released by the barrier ending chunk c-1
    mbar_wait(smem_u32(&full[buf]), (uint32_t)(c / H2_STAGES) & 1u);
    const H2Stage &b = st[buf];
    if (warp < NW) {
#pragma unroll 4
      for (int kk = 0; kk < H2_KC; kk += 4) {
        float4 x[NS];
#pragma unroll
        for (int i = 0; i < NS; i++) x[i] = *(const float4 *)&b.xs[row0 + i][kk];
        const float2 w0 = *(const float2 *)&b.ws[kk][o2], w1 = *(const float2 *)&b.ws[kk + 1][o2];
        const float2 w2 = *(const float2 *)&b.ws[kk + 2][o2], w3 = *(const float2 *)&b.ws[kk + 3][o2];
#pragma unroll
        for (int i = 0; i < NS; i++) { acc[i][0] = fmaf(w0.x, x[i].x, acc[i][0]); acc[i][1] = fmaf(w0.y, x[i].x, acc[i][1]); }
#pragma unroll
        for (int i = 0; i < NS; i++) { acc[i][0] = fmaf(w1.x, x[i].y, acc[i][0]); acc[i][1] = fmaf(w1.y, x[i].y, acc[i][1]); }
#pragma unroll
        for (int i = 0; i < NS; i++) { acc[i][0] = fmaf(w2.x, x[i].z, acc[i][0]); acc[i][1] = fmaf(w2.y, x[i].z, acc[i][1]); }
#pragma unroll
        for (int i = 0; i < NS; i++) { acc[i][0] = fmaf(w3.x, x[i].w, acc[i][0]); acc[i][1] = fmaf(w3.y, x[i].w, acc[i][1]); }
      }
    } else {
#pragma unroll 4
      for (int kk = 0; kk < H2_KC; kk += 4) {
        const float4 x = *(const float4 *)&b.xs[lane < TS ? lane : 0][kk], w = *(const float4 *)&wv_all[c * H2_KC + kk];
        y = y + w.x * x.x; y = y + w.y * x.y; y = y + w.z * x.z; y = y + w.w * x.w;
      }
    }
    __syncthreads();   // everyone is done with this stage before the producer refills it
  }
  if (warp < NW) {
    const float b0 = m.dense_out.bias[o2], b1 = m.dense_out.bias[o2 + 1];
#pragma unroll
    for (int i = 0; i < NS; i++) {
      const int s = s0 + row0 + i;
      if (s < S) *(float2 *)&gains[(size_t)s * NB_GAINS + o2] = make_float2(act_sigmoid(acc[i][0] + b0), act_sigmoid(acc[i][1] + b1));
    }
  } else {
    const int s = s0 + lane;
    if (lane < TS && s < S) {
      const float v = silence[s] ? 0.f : act_sigmoid(y + m.vad_dense.bias[0]);
      vad[s] = v;
      if (vad_user) vad_user[(size_t)s * vad_stride] = v;
    }
  }
}
