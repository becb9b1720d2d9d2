// gru_tc.cuh -- the int8 tensor-core kernels of the network on Hopper (wgmma): one GRU layer or conv2 per launch.
//
//   D_in [M x 3U] = Xu8[M x K] . Wi_slice^T      (u8 x s8 -> s32, wgmma.mma_async m64nNk32)
//   D_rec[M x 3U] = Hu8[M x K] . Wr_slice^T      3U = {z, r, n} x U units, K = gru (384)
//
// Operands arrive by TMA (cp.async.bulk.tensor, SWIZZLE_128B, K-major) straight from the u8 mirrors of the
// activations / the pre-permuted s8 weights, and wgmma reads them through shared-memory matrix descriptors.  The s32
// accumulators live in the registers of the warpgroup that issued the MMAs; that warpgroup applies, in registers,
// exactly the arithmetic of the reference (compute_linear + compute_generic_gru, src/nnet_arch.h:130-162,
// src/nnet.c:65-94): (float)acc*scale + subias, fma(diag,h,.), sigmoid/sigmoid/tanh, h' = z*h + (1-z)*n, then stores
// h' as fp32 AND as the u8 operand of the next consumer.  The integer accumulators are exact, so these kernels are
// bit-identical to the dp4a kernels k_gru / k_conv2.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "rnn_kernels.cuh"

#define TC_M 128          // streams per CTA tile: two 64-row wgmma halves
#define TC_UNITS 32       // hidden units per CTA of k_gru_tc
#define TC_N (3 * TC_UNITS)  // wgmma N of k_gru_tc = 96
#define TC_KATOM 128      // bytes of K per 128B-swizzle atom
#define TC_HALF_BYTES (64 * TC_KATOM)   // byte offset of rows 64..127 inside an A atom

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a lost transaction (bad tensor map / byte count) becomes a trap -> CUDA error on the
// host instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// K-major, 128B-swizzled operand tile: rows of 128 bytes, 8-row groups 1024 B apart (wgmma matrix descriptor:
// start>>4 | LBO(unused by this layout, 1)<<16 | SBO(1024>>4)<<32 | SWIZZLE_128B(1)<<62).  The tile base is
// 1024-byte aligned, so the descriptor's base offset is 0; +2 in the start field advances K by 32 bytes.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// after wgmma_wait_all(): keeps every use of the accumulators behind the wait
template <int R>
__device__ __forceinline__ void wgmma_hold(int (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 32 B] . B[N x 32 B]^T, u8 x s8 -> s32; acc = 0 overwrites D
__device__ __forceinline__ void wgmma_i8(int (&d)[8], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
      : "l"(a), "l"(b), "r"(acc)
      : "memory");
}
__device__ __forceinline__ void wgmma_i8(int (&d)[24], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
        "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
      : "l"(a), "l"(b), "r"(acc)
      : "memory");
}
__device__ __forceinline__ void wgmma_i8(int (&d)[48], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
      "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
        "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]),
        "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
      : "l"(a), "l"(b), "r"(acc)
      : "memory");
}
// d = A[64 rows x K] . B[N rows x K]^T over `natoms` 128-byte K atoms (A atoms a_stride, B atoms b_stride bytes apart),
// issued by the whole warpgroup; the caller fences before and commits / waits after
// wgmma_chain unrolls the chain for its atom count (1..8, K <= 1024): with a run-time loop ptxas serialises the wgmma of
// the chain and inserts warpgroup fences of its own (C7515 / C7520 in `build.py -v`).  k_net keeps the run-time loop
// (wgmma_chain_rt): a 544-thread CTA gets at most 96 registers per thread, and the unrolled chains of its four layer
// shapes raise its spills from ~0.3 KB to ~1 KB of loads per thread.
template <int NA, int R>
__device__ __forceinline__ void wgmma_chain_n(int (&d)[R], uint32_t A, int a_stride, uint32_t B, int b_stride) {
#pragma unroll
  for (int a = 0; a < NA; a++) {
    const uint64_t ad = wgmma_desc_sw128(A + a * a_stride), bd = wgmma_desc_sw128(B + a * b_stride);
#pragma unroll
    for (int k = 0; k < TC_KATOM / 32; k++) wgmma_i8(d, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (a | k) ? 1 : 0);
  }
}
template <int R>
__device__ __forceinline__ void wgmma_chain_rt(int (&d)[R], uint32_t A, int a_stride, uint32_t B, int b_stride, int natoms) {
  for (int a = 0; a < natoms; a++) {
    const uint64_t ad = wgmma_desc_sw128(A + a * a_stride), bd = wgmma_desc_sw128(B + a * b_stride);
#pragma unroll
    for (int k = 0; k < TC_KATOM / 32; k++) wgmma_i8(d, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (a | k) ? 1 : 0);
  }
}
template <int R>
__device__ __forceinline__ void wgmma_chain(int (&d)[R], uint32_t A, int a_stride, uint32_t B, int b_stride, int natoms) {
  switch (natoms) {
    case 1: wgmma_chain_n<1>(d, A, a_stride, B, b_stride); break;
    case 2: wgmma_chain_n<2>(d, A, a_stride, B, b_stride); break;
    case 3: wgmma_chain_n<3>(d, A, a_stride, B, b_stride); break;
    case 4: wgmma_chain_n<4>(d, A, a_stride, B, b_stride); break;
    case 5: wgmma_chain_n<5>(d, A, a_stride, B, b_stride); break;
    case 6: wgmma_chain_n<6>(d, A, a_stride, B, b_stride); break;
    case 7: wgmma_chain_n<7>(d, A, a_stride, B, b_stride); break;
    default: wgmma_chain_n<8>(d, A, a_stride, B, b_stride); break;
  }
}

// Accumulator fragment of wgmma m64nNk32 (PTX ISA, "Register fragments", matrix D): thread `lane` of warp w of the
// warpgroup holds d[4 j + 2 h + e] = D[16 (w % 4) + lane / 4 + 8 h][8 j + 2 (lane % 4) + e] for every 8-column block j.
// Of a block of U units per gate (the N columns are z | r | n, U each) a thread therefore owns the rows
// 16 (w % 4) + lane / 4 + {0, 8} and, in each, the P = U / 4 units frag_unit(q): neighbour pairs 8 i + 2 (lane % 4) + {0, 1}.
__device__ __forceinline__ int frag_unit(int q) { return 8 * (q >> 1) + 2 * (int)(threadIdx.x & 3) + (q & 1); }
template <int U>
__device__ __forceinline__ int frag_idx(int g, int h, int q) { return 4 * ((U / 8) * g + (q >> 1)) + 2 * h + (q & 1); }
__device__ __forceinline__ int frag_row(int warp) { return 16 * (warp & 3) + ((int)(threadIdx.x & 31) >> 2); }

// fp32 values of a thread's P units of one row (row -> unit 0 of the tile; pairs of neighbours: 8-byte loads)
template <int P>
__device__ __forceinline__ void frag_load_row(const float *row, float (&v)[P]) {
#pragma unroll
  for (int k = 0; k < P / 2; k++) {
    const float2 t = __ldg((const float2 *)&row[frag_unit(2 * k)]);
    v[2 * k] = t.x; v[2 * k + 1] = t.y;
  }
}
// the fp32 outputs and their u8 operand mirror
template <int P>
__device__ __forceinline__ void frag_store_row(float *row, uint8_t *row_u8, const float (&v)[P]) {
#pragma unroll
  for (int k = 0; k < P / 2; k++) {
    const int u = frag_unit(2 * k);
    *(float2 *)&row[u] = make_float2(v[2 * k], v[2 * k + 1]);
    *(uint16_t *)&row_u8[u] = (uint16_t)(quant_u8(v[2 * k]) | (quant_u8(v[2 * k + 1]) << 8));
  }
}
// GRU update of row h (0 / 1) of a thread's fragment of a U-unit tile from the input (ai) and recurrent (ar)
// accumulators; prm = the tile's epilogue parameter records [U][16] (DevLayerQ::packed): {sc_i, sb_i, sc_r, sb_r} for
// z, r, n, then {diag_z, diag_r, diag_n, 0}
template <int U>
__device__ __forceinline__ void gru_frag(const int (&ai)[3 * U / 2], const int (&ar)[3 * U / 2], const float *prm, int h,
                                         const float (&hold)[U / 4], float (&out)[U / 4]) {
  constexpr int P = U / 4;
  float zi[P], ri[P], ni[P], zr[P], rr[P], nr[P];
#pragma unroll
  for (int q = 0; q < P; q++) {
    const float *pu = prm + 16 * frag_unit(q);
    const float x = hold[q];
    const float4 pz = *(const float4 *)&pu[0], pr = *(const float4 *)&pu[4];
    const float4 pn = *(const float4 *)&pu[8], pd = *(const float4 *)&pu[12];
    zi[q] = (float)ai[frag_idx<U>(0, h, q)] * pz.x + pz.y;
    ri[q] = (float)ai[frag_idx<U>(1, h, q)] * pr.x + pr.y;
    ni[q] = (float)ai[frag_idx<U>(2, h, q)] * pn.x + pn.y;
    zr[q] = fmaf(pd.x, x, (float)ar[frag_idx<U>(0, h, q)] * pz.z + pz.w);
    rr[q] = fmaf(pd.y, x, (float)ar[frag_idx<U>(1, h, q)] * pr.z + pr.w);
    nr[q] = fmaf(pd.z, x, (float)ar[frag_idx<U>(2, h, q)] * pn.z + pn.w);
  }
  gru_units<P>(zi, ri, ni, zr, rr, nr, hold, out);
}
// conv2 output (tanh(acc * scale + subias)) of row h of a thread's fragment of a 16-unit slice; scale / subias -> unit 0
__device__ __forceinline__ void conv_frag(const int (&acc)[8], const float *scale, const float *subias, int h, float (&out)[4]) {
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int u = frag_unit(q);
    out[q] = (float)acc[frag_idx<16>(0, h, q)] * scale[u] + subias[u];
  }
  if (fabsf(out[0]) < ACT_FAST_LIMIT && fabsf(out[1]) < ACT_FAST_LIMIT && fabsf(out[2]) < ACT_FAST_LIMIT && fabsf(out[3]) < ACT_FAST_LIMIT) {
#pragma unroll
    for (int q = 0; q < 4; q++) out[q] = act_tanh_inrange(out[q]);
  } else {
#pragma unroll
    for (int q = 0; q < 4; q++) out[q] = act_tanh(out[q]);
  }
}

struct GruTcMaps {
  CUtensorMap x, h, wi, wr;   // x,h: u8 [S][K]; wi,wr: s8 [(K/units slices) * 3 * units][K] permuted
};

// ================================================================================================
// k_gru_tc -- one GRU layer, one tile of 128 streams x 32 units per CTA (cross-check of k_tc2).
// grid = (ceil(S/128), gru/32), block = 160: warps 0..3 = the warpgroup that issues the MMAs (M64 x N96 per matrix,
// the two 64-row halves of the tile in turn) and runs the epilogue; warp 4 = TMA producer.
// dynamic smem = gru_tc_smem_bytes(gru), 1 CTA / SM.
// ================================================================================================
// smem: A tiles (X, H): 2 x (K/128) x 16 KB ; B tiles (Wi, Wr): 2 x (K/128) x 12 KB ; parameters ; barrier
#define TC_A_ATOM_BYTES (TC_M * TC_KATOM)     // 16384
#define TC_B_ATOM_BYTES (TC_N * TC_KATOM)     // 12288
__host__ __device__ constexpr int gru_tc_smem_bytes(int gru) {
  return 1024 /*align slack*/ + 2 * (gru / TC_KATOM) * (TC_A_ATOM_BYTES + TC_B_ATOM_BYTES) + 16 * TC_UNITS * 4 + 64;
}

__global__ void __launch_bounds__(160, 1)
k_gru_tc(int S, int gru, const __grid_constant__ GruTcMaps maps, DevLayerQ wi, DevLayerQ wr,
         const float *__restrict__ h_old, float *__restrict__ h_new, uint8_t *__restrict__ h_new_u8,
         const int *__restrict__ silence) {
  (void)wi;   // its epilogue parameters are part of the layer's packed records (wr.packed)
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * TC_M, j0 = blockIdx.y * TC_UNITS, natoms = gru / TC_KATOM;
  // 1024-byte aligned operand area (SWIZZLE_128B requirement); plain pointer arithmetic on the shared
  // array keeps the address space known to the compiler (LDS/STS instead of generic loads)
  uint8_t *base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t *sAx = base, *sAh = sAx + natoms * TC_A_ATOM_BYTES;
  uint8_t *sBi = sAh + natoms * TC_A_ATOM_BYTES, *sBr = sBi + natoms * TC_B_ATOM_BYTES;
  float *prm = (float *)(sBr + natoms * TC_B_ATOM_BYTES);       // [32][16]: packed records of the tile's units
  uint64_t *bars = (uint64_t *)(prm + 16 * TC_UNITS);           // [0] operands landed
  const uint32_t bar_full = smem_u32(&bars[0]);

  if (tid == 0) {
    mbar_init(bar_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp < 4)
    for (int c = tid; c < 4 * TC_UNITS; c += 128) cp_async16(prm + 4 * c, wr.packed + (size_t)j0 * 16 + 4 * c, true);
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      // ---- TMA producer: everything this CTA needs, one transaction barrier ----
      mbar_expect_tx(bar_full, (uint32_t)(2 * natoms * (TC_A_ATOM_BYTES + TC_B_ATOM_BYTES)));
      for (int a = 0; a < natoms; a++) {
        tma_load_2d(smem_u32(sAx + a * TC_A_ATOM_BYTES), &maps.x, bar_full, a * TC_KATOM, m0);
        tma_load_2d(smem_u32(sBi + a * TC_B_ATOM_BYTES), &maps.wi, bar_full, a * TC_KATOM, blockIdx.y * TC_N);
      }
      for (int a = 0; a < natoms; a++) {
        tma_load_2d(smem_u32(sAh + a * TC_A_ATOM_BYTES), &maps.h, bar_full, a * TC_KATOM, m0);
        tma_load_2d(smem_u32(sBr + a * TC_B_ATOM_BYTES), &maps.wr, bar_full, a * TC_KATOM, blockIdx.y * TC_N);
      }
    }
    return;
  }
  mbar_wait(bar_full, 0);
  for (int mh = 0; mh < 2; mh++) {
    const int r0 = m0 + 64 * mh + frag_row(warp);
    bool live[2], silent[2];
    float hold[2][TC_UNITS / 4];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = r0 + 8 * h;
      live[h] = row < S;
      silent[h] = live[h] ? silence[row] != 0 : true;
      if (live[h]) frag_load_row(h_old + (size_t)row * gru + j0, hold[h]);
      else
#pragma unroll
        for (int q = 0; q < TC_UNITS / 4; q++) hold[h][q] = 0.f;
    }
    int ai[3 * TC_UNITS / 2], ar[3 * TC_UNITS / 2];
#pragma unroll
    for (int i = 0; i < 3 * TC_UNITS / 2; i++) ai[i] = ar[i] = 0;
    wgmma_fence();
    wgmma_chain(ai, smem_u32(sAx) + mh * TC_HALF_BYTES, TC_A_ATOM_BYTES, smem_u32(sBi), TC_B_ATOM_BYTES, natoms);
    wgmma_chain(ar, smem_u32(sAh) + mh * TC_HALF_BYTES, TC_A_ATOM_BYTES, smem_u32(sBr), TC_B_ATOM_BYTES, natoms);
    wgmma_commit();
    wgmma_wait_all();
    wgmma_hold(ai); wgmma_hold(ar);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float outv[TC_UNITS / 4];
      if (silent[h]) {
#pragma unroll
        for (int q = 0; q < TC_UNITS / 4; q++) outv[q] = hold[h][q];
      } else {
        gru_frag<TC_UNITS>(ai, ar, prm, h, hold[h], outv);
      }
      const size_t row = (size_t)(r0 + 8 * h);
      if (live[h]) frag_store_row(h_new + row * gru + j0, h_new_u8 + row * gru + j0, outv);
    }
  }
}

// ================================================================================================
// k_tc2<kGru> -- persistent, warp-specialised tensor-core kernel (the default int8 path).
//
//   kGru = true : one GRU layer (k_gru_tc2).   kGru = false: conv2 (k_conv2_tc), a single GEMM + tanh.
//
// CTA = 128 streams x (N/4) output units, processed as slices of 16 units; the weight slices stream through a
// TC2_STAGES-deep TMA ring (see ring_stage below):
//     warp 16 (one elected thread): TMA producer
//     warps 0..15 = four warpgroups : warpgroup g takes rows 64 (g & 1) .. + 64 of the slices s with s % 2 == g >> 1,
//                                     issues their MMAs and runs their epilogue
// so that the MMAs of one slice run beside the epilogue of the other warpgroup pair's slice.  The u8 activation tiles
// (128 x K; GRU: Xu8 and Hu8) are loaded once per CTA and stay resident.  Per slice and matrix one wgmma chain of
// K/32 instructions, M64 x N48 (GRU: z|r|n of 16 units) or N16 (conv2), accumulators in registers.
// Same arithmetic as the dp4a kernels k_gru / k_conv2: bit-identical results.
// grid = (ceil(S/128), 4), block = 544, 1 CTA / SM.
// ================================================================================================
#define P_SLICE 16
// Weight rings: job j (a slice) is consumed by warpgroup pair j & 1, and each pair owns half of the stages, which it
// uses in turn.  So every load into a stage is consumed by the same pair, in the order the loads were issued, and the
// phase parity a consumer waits for always names the load it wants: a stage shared by both pairs could be waited on
// while the other pair's earlier load into it is still in flight (TMA completions are not ordered), and the wait would
// pass on the stale phase.  Stage counts are therefore even.  A pair releases its stage when its MMAs have retired,
// long before its epilogue ends, so one stage per pair keeps the producer ahead of the MMAs.
#ifndef P_STAGES
#define P_STAGES 2                        // weight ring of the fused network kernel (net_kernel.cuh)
#endif
#ifndef TC2_STAGES
#define TC2_STAGES 2                      // weight ring of the per-layer kernels
#endif
static_assert(P_STAGES % 2 == 0 && P_STAGES >= 2 && P_STAGES <= 4, "P_STAGES: 2 or 4 (one or two stages per warpgroup pair)");
static_assert(TC2_STAGES % 2 == 0 && TC2_STAGES >= 2 && TC2_STAGES <= 4, "TC2_STAGES: 2 or 4 (one or two stages per warpgroup pair)");
// stage of job j in a ring of `stages`, and how many earlier jobs used that stage (its phase count)
__host__ __device__ constexpr int ring_stage(int j, int stages) { return (j & 1) * (stages / 2) + (j >> 1) % (stages / 2); }
__host__ __device__ constexpr int ring_use(int j, int stages) { return (j >> 1) / (stages / 2); }
// L2 prefetch of the CTA's old-state rows at kernel start (no registers held): the state was written a whole frame ago
// and has left the L2 at large batch sizes, so the per-slice gathers of the epilogue otherwise wait on HBM.
#ifndef TC2_H_L2PF
#define TC2_H_L2PF 1
#endif

template <bool kGru> struct TcCfg {
  static constexpr int kMats = kGru ? 2 : 1;                 // GEMMs per slice (input, recurrent)
  static constexpr int kN = kGru ? 3 * P_SLICE : P_SLICE;    // wgmma N: 48 / 16
  static constexpr int kBAtom = kN * TC_KATOM;               // bytes of one weight atom: 6144 / 2048
  static constexpr int kPrm = kGru ? 16 : 2;                 // epilogue parameters per unit (GRU: 4 float4, see below)
  static constexpr int kAcc = kN / 2;                        // accumulator registers per thread and matrix: 24 / 8
};
template <bool kGru>
__host__ __device__ constexpr int tc2_smem_bytes(int K, int N) {
  return 1024 + TcCfg<kGru>::kMats * (K / TC_KATOM) * TC_A_ATOM_BYTES +
         TC2_STAGES * TcCfg<kGru>::kMats * (K / TC_KATOM) * TcCfg<kGru>::kBAtom + TcCfg<kGru>::kPrm * (N / 4) * 4 + 16 * 8 + 64;
}

#define P_EPI_WARPS 16                    // MMA + epilogue warps: four warpgroups
#define P_PAIR_WARPS 8                    // warps of the warpgroup pair that consumes one slice
#define P_UPT (P_SLICE / 4)               // units per thread and row of a slice: 4
#define P_THREADS (32 * (P_EPI_WARPS + 1))

// K = contraction length = bytes of one (zero-weight padded) activation row, a multiple of 128; N = number of output
// units (gru, a multiple of 64); ldo = row stride of the u8 output mirror (the padded K of its consumer).
// GRU : maps.x/h = Xu8/Hu8 [S][K]; maps.wi/wr = s8 [(N/16) x 48][K];  out = h_new (+u8), aux = h_old
// conv: maps.x = conv2 input u8 [S][K]; maps.wi = s8 [N][K] (unit-major); out = conv2_out (+u8)
template <bool kGru>
__global__ void __launch_bounds__(P_THREADS, 1)
k_tc2(int S, int K, int N, int ldo, const __grid_constant__ GruTcMaps maps, DevLayerQ wi, DevLayerQ wr,
      const float *__restrict__ h_old, float *__restrict__ out_f32, uint8_t *__restrict__ out_u8,
      const int *__restrict__ silence) {
  using C = TcCfg<kGru>;
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int natoms = K / TC_KATOM, upc = N / 4, nslice = upc / P_SLICE;   // units / slices per CTA
  const int m0 = blockIdx.x * TC_M, jq = blockIdx.y * upc;
  // 1024-byte aligned operand area; pointer arithmetic on the shared array keeps the address space
  // known to the compiler (LDS instead of generic loads for the epilogue parameters)
  uint8_t *base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t *sAx = base, *sAh = sAx + natoms * TC_A_ATOM_BYTES;
  uint8_t *sB = sAx + C::kMats * natoms * TC_A_ATOM_BYTES;
  const int stage_bytes = C::kMats * natoms * C::kBAtom;
  float *prm = (float *)(sB + TC2_STAGES * stage_bytes);            // [kPrm][upc]
  uint64_t *bars = (uint64_t *)(prm + C::kPrm * upc);
  const uint32_t bar_a = smem_u32(&bars[0]);
  auto bar_bfull = [&](int i) { return smem_u32(&bars[1 + i]); };
  auto bar_bempty = [&](int i) { return smem_u32(&bars[8 + i]); };

  pdl_trigger();
  auto load_B = [&](int s) {
    const int st = ring_stage(s, TC2_STAGES);
    uint8_t *dst = sB + st * stage_bytes;
    const int row = (blockIdx.y * nslice + s) * C::kN;
    mbar_expect_tx(bar_bfull(st), (uint32_t)stage_bytes);
    for (int a = 0; a < natoms; a++) {
      tma_load_2d(smem_u32(dst + a * C::kBAtom), &maps.wi, bar_bfull(st), a * TC_KATOM, row);
      if (kGru) tma_load_2d(smem_u32(dst + (natoms + a) * C::kBAtom), &maps.wr, bar_bfull(st), a * TC_KATOM, row);
    }
  };
  // The producer thread initialises the barriers ITSELF and starts the weight and operand-tile loads right away:
  // they overlap the (scattered) parameter staging below instead of following it (the other threads touch the
  // barriers only after the __syncthreads that ends the prologue).
  if (warp == P_EPI_WARPS && lane == 0) {
    mbar_init(bar_a, 1);
    for (int i = 0; i < TC2_STAGES; i++) { mbar_init(bar_bfull(i), 1); mbar_init(bar_bempty(i), P_PAIR_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // first what the first slice needs (its weights, then the operand tiles), then the other weight stages: every CTA
    // of the grid starts here at the same time and the burst is bound by L2 bandwidth
    load_B(0);                                                     // weights: independent of the previous kernel
    pdl_wait();                                                    // activations of this frame are complete
    mbar_expect_tx(bar_a, (uint32_t)(C::kMats * natoms * TC_A_ATOM_BYTES));
    for (int a = 0; a < natoms; a++) {
      tma_load_2d(smem_u32(sAx + a * TC_A_ATOM_BYTES), &maps.x, bar_a, a * TC_KATOM, m0);
      if (kGru) tma_load_2d(smem_u32(sAh + a * TC_A_ATOM_BYTES), &maps.h, bar_a, a * TC_KATOM, m0);
    }
    for (int s = 1; s < TC2_STAGES && s < nslice; s++) load_B(s);
  }
  if (kGru) {
    // per unit u: {sc_i, sb_i, sc_r, sb_r} for z, r, n, then {diag_z, diag_r, diag_n, 0} (four LDS.128 in the epilogue):
    // this CTA's slice of the layer's packed records (DevLayerQ::packed) is contiguous -- 16-byte asynchronous copies
    // issued by the MMA warps, which wait for them only right before their first slice
    const float *src = wr.packed + (size_t)jq * 16;
    if (warp < P_EPI_WARPS)
      for (int c = tid; c < 4 * upc; c += 32 * P_EPI_WARPS) cp_async16(prm + 4 * c, src + 4 * c, true);
    asm volatile("cp.async.commit_group;" ::: "memory");
  } else {
    for (int i = tid; i < C::kPrm * upc; i += blockDim.x) prm[i] = (i < upc ? wi.scale : wi.subias)[jq + i % upc];
  }
  __syncthreads();

  if (warp == P_EPI_WARPS) {
    if (lane == 0)
      for (int s = TC2_STAGES; s < nslice; s++) {   // refill a stage once the pair that read it has released it
        mbar_wait(bar_bempty(ring_stage(s, TC2_STAGES)), (uint32_t)((ring_use(s, TC2_STAGES) - 1) & 1));
        load_B(s);
      }
    return;
  }
  const int pair = warp / P_PAIR_WARPS, mh = (warp >> 2) & 1;
  const int r0 = m0 + 64 * mh + frag_row(warp);
  bool live[2], silent[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int row = r0 + 8 * h;
    live[h] = row < S;
    silent[h] = live[h] ? silence[row] != 0 : true;
    // the row's upc floats = upc / 32 lines of 128 bytes, shared out over the 8 threads of both pairs that own the row
    if (TC2_H_L2PF && kGru && live[h])
      for (int l = 4 * pair + (lane & 3); l * 32 < upc; l += 8)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(&h_old[(size_t)row * N + jq + l * 32]) : "memory");
  }
  if (kGru) {   // the parameter records requested in the prologue: own copies landed, then visible to all MMA warps
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    asm volatile("bar.sync 1, %0;" ::"n"(32 * P_EPI_WARPS) : "memory");
  }
  mbar_wait(bar_a, 0);
  const uint32_t aX = smem_u32(sAx) + mh * TC_HALF_BYTES, aH = smem_u32(sAh) + mh * TC_HALF_BYTES;
  for (int s = pair; s < nslice; s += 2) {
    const int st = ring_stage(s, TC2_STAGES), ub = s * P_SLICE;   // ub: first unit of the slice inside this CTA's quarter
    float hold[2][P_UPT];
#pragma unroll
    for (int h = 0; h < 2; h++) {   // old state: in flight while the MMAs run
      if (kGru && live[h]) frag_load_row(h_old + (size_t)(r0 + 8 * h) * N + jq + ub, hold[h]);
      else
#pragma unroll
        for (int q = 0; q < P_UPT; q++) hold[h][q] = 0.f;
    }
    int ai[C::kAcc], ar[C::kAcc];
#pragma unroll
    for (int i = 0; i < C::kAcc; i++) ai[i] = ar[i] = 0;
    mbar_wait(bar_bfull(st), (uint32_t)(ring_use(s, TC2_STAGES) & 1));
    const uint32_t Bs = smem_u32(sB + st * stage_bytes);
    wgmma_fence();
    wgmma_chain(ai, aX, TC_A_ATOM_BYTES, Bs, C::kBAtom, natoms);
    if (kGru) wgmma_chain(ar, aH, TC_A_ATOM_BYTES, Bs + natoms * C::kBAtom, C::kBAtom, natoms);
    wgmma_commit();
    wgmma_wait_all();
    wgmma_hold(ai); wgmma_hold(ar);
    // the weight stage has been read: hand it back to the producer
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_bempty(st));
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float outv[P_UPT];
      if constexpr (kGru) {
        if (silent[h]) {
#pragma unroll
          for (int q = 0; q < P_UPT; q++) outv[q] = hold[h][q];
        } else {
          gru_frag<P_SLICE>(ai, ar, prm + 16 * ub, h, hold[h], outv);
        }
      } else {
        conv_frag(ai, prm + ub, prm + upc + ub, h, outv);
      }
      const size_t row = (size_t)(r0 + 8 * h);
      if (live[h]) frag_store_row(out_f32 + row * N + jq + ub, out_u8 + row * ldo + jq + ub, outv);
    }
  }
}
