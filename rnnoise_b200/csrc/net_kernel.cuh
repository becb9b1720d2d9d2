// net_kernel.cuh -- conv1 -> conv2 -> GRU1 -> GRU2 -> GRU3 of compute_rnn() (reference src/rnn.c:44-60) as ONE persistent
// wgmma kernel over a 4-CTA thread-block cluster per 128-stream tile (the default network path for small batches; the
// per-layer kernels k_tc2<> of gru_tc.cuh run the same arithmetic one layer per launch).
//
//   cluster = 4 CTAs = one tile of 128 streams; CTA r of the cluster owns output units [r*N/4, (r+1)*N/4) of
//   EVERY layer.  Per layer a CTA needs the whole u8 activation rows of the previous layer (K = N bytes per
//   stream): each CTA writes its unit quarter (fp32 state + u8 operand mirror) to global memory, the cluster
//   synchronises (barrier.cluster release/acquire + proxy fence), and every CTA TMA-loads the full 128 x K tile
//   back from L2.  The recurrent operand Hu8 of the NEXT layer does not depend on this frame, so its TMA load is
//   issued as soon as the current layer's MMAs have retired and hides behind the epilogue tail; the weight-slice
//   ring (one stage per warpgroup pair) simply runs on across layer boundaries, so the weights of the next layer's first slices are
//   already in shared memory when its activations arrive.
//
//   conv1 (fp32, 195 -> cond, one sequential FMA chain per output: nnet.c:113-123, sgemv vec_avx.h:672) runs as a
//   prologue on the epilogue warps while the producer prefetches weights: CTA r computes it for streams
//   [32 r, 32 r + 32) of the tile (thread = output x 8 streams, inputs transposed in shared memory), updates the
//   conv1 memory and conv2's u8 operand rows in global memory, and the cluster barrier that starts conv2 publishes
//   them.  (k_conv1 of rnn_kernels.cuh is the stand-alone cross-check.)
//
//   warp 16 (one elected thread)  : TMA producer                                          (as in k_tc2)
//   warps 0..15 = four warpgroups : MMAs + epilogue; the slices of all layers are numbered in one sequence (jobs) and
//                                   warpgroup g takes rows 64 (g & 1) .. + 64 of the jobs j with j % 2 == g >> 1
//
// Against one launch per layer this removes four kernel boundaries (drain, launch latency, barrier/parameter
// prologue, cold TMA pipeline) per frame and lane.  Arithmetic: identical to k_tc2 / the dp4a kernels, bit for bit
// (exact s32 accumulators; (float)acc*scale + subias; fma(diag,h,.); Pade sigmoid/tanh; h' = z*h + (1-z)*n).
// grid = (ceil(S/128), R), cluster (1,R,1) with R = 4 or 8, block = 544, dynamic smem = net_smem_bytes(), 1 CTA / SM.
#pragma once
#include "gru_tc.cuh"

#define NET_LAYERS 4   // conv2 + 3 GRU

struct NetMaps {       // TMA descriptors of one frame parity
  CUtensorMap x[NET_LAYERS], h[NET_LAYERS], wi[NET_LAYERS], wr[NET_LAYERS];   // h / wr unused for layer 0 (conv2)
};
struct NetPtrs {
  const float *scale_i[NET_LAYERS], *subias_i[NET_LAYERS];   // input matrix (conv2: the only matrix)
  const float *scale_r[NET_LAYERS], *subias_r[NET_LAYERS], *diag[NET_LAYERS];
  const float *packed[NET_LAYERS];    // GRU layers: DevLayerQ::packed, [N][16] epilogue parameter records
  const float *h_old[NET_LAYERS];     // fp32 state of the previous frame (GRU layers)
  float *out_f32[NET_LAYERS];         // conv2_out / new fp32 state
  uint8_t *out_u8[NET_LAYERS];        // their u8 operand mirrors
  // conv1 prologue (conv1_w == nullptr: conv2's operand rows were prepared by k_conv1)
  const float *conv1_w, *conv1_b;     // [195][cond], [cond]
  const float *features;              // [S][65] of this frame
  float *conv1_state;                 // [S][130]
  uint8_t *c2in;                      // [S][Kc] conv2 operand rows: [memory (2 x cond) | newest (cond) | pad]
  int cond;
};
#define NET_C1_IN (3 * NB_FEAT)       // 195

__host__ __device__ constexpr int net_stage_bytes(int K) { return 2 * (K / TC_KATOM) * (3 * P_SLICE * TC_KATOM); }
__host__ __device__ constexpr int net_prm_floats(int N) { return (2 + 3 * 16) * (N / 4); }   // sized for the smallest cluster (4)
__host__ __device__ constexpr int net_smem_bytes(int Kc, int Kn, int N) {
  // A tiles: X (max(Kc, Kn) bytes per row) + H (Kn); B ring; parameters of all layers; barriers
  return 1024 + ((Kc > Kn ? Kc : Kn) / TC_KATOM + Kn / TC_KATOM) * TC_A_ATOM_BYTES + P_STAGES * net_stage_bytes(Kn) +
         net_prm_floats(N) * 4 + 24 * 8 + 64;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Kc = conv2's contraction length (3 * cond) and Kn = the GRU layers' (gru), both padded up to multiples of 128 with
// zero weights; N = gru (a multiple of 64).  Kn is also the row stride of every u8 activation mirror.
// The cluster size R = gridDim.y (4 or 8, set by the launch attribute) splits every layer's units R ways: R = 8 halves
// each CTA's share (and the kernel's latency) at the price of twice the SMs per tile.
__global__ void __launch_bounds__(P_THREADS, 1)
k_net(int S, int Kc, int Kn, int N, const __grid_constant__ NetMaps maps, const __grid_constant__ NetPtrs p, const int *__restrict__ silence) {
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = (int)gridDim.y, upc = N / R, nslice = upc / P_SLICE;   // units / slices per CTA
  const int atoms_c = Kc / TC_KATOM, atoms_n = Kn / TC_KATOM, atoms_x = atoms_c > atoms_n ? atoms_c : atoms_n;
  const int m0 = blockIdx.x * TC_M, jq = blockIdx.y * upc;
  uint8_t *base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t *sAx = base, *sAh = sAx + atoms_x * TC_A_ATOM_BYTES;
  uint8_t *sB = sAh + atoms_n * TC_A_ATOM_BYTES;
  const int stage_bytes = net_stage_bytes(Kn);
  float *prm = (float *)(sB + P_STAGES * stage_bytes);   // conv: [2][upc]; then per GRU layer [upc][16]
  uint64_t *bars = (uint64_t *)(prm + net_prm_floats(N));
  const uint32_t bar_x = smem_u32(&bars[0]), bar_h = smem_u32(&bars[1]), bar_adone = smem_u32(&bars[2]);
  auto bar_bfull = [&](int i) { return smem_u32(&bars[4 + i]); };
  auto bar_bempty = [&](int i) { return smem_u32(&bars[8 + i]); };

  if (tid == 0) {
    // bar_adone: every MMA warp has finished reading the activation tiles of the current layer
    mbar_init(bar_x, 1); mbar_init(bar_h, 1); mbar_init(bar_adone, P_EPI_WARPS);
    for (int i = 0; i < P_STAGES; i++) { mbar_init(bar_bfull(i), 1); mbar_init(bar_bempty(i), P_PAIR_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // epilogue parameters of this CTA's unit quarter, all layers
  for (int i = tid; i < 2 * upc; i += blockDim.x) prm[i] = (i < upc ? p.scale_i[0] : p.subias_i[0])[jq + i % upc];
  // GRU layers: this CTA's unit slice of the packed parameter records, contiguous in memory and in shared memory:
  // 16-byte asynchronous copies, all in flight together (six dependent scattered loads per thread before)
  for (int L = 1; L < NET_LAYERS; L++) {
    float *pl = prm + 2 * upc + (L - 1) * 16 * upc;
    const float *src = p.packed[L] + (size_t)jq * 16;
    for (int c = tid; c < 4 * upc; c += blockDim.x) cp_async16(pl + 4 * c, src + 4 * c, true);
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  if (p.conv1_w && warp < P_EPI_WARPS) {
    // ---- conv1 prologue for streams [m0 + 32 r, + 32), r = this CTA's rank; the X tile region is still free ----
    float *tmpT = (float *)sAx;                      // [195][32]: input j of the 32 streams (conflict-free, LDS.128 broadcast)
    const int cond = p.cond, W = cond / 4, nrow = TC_M / R, r0 = m0 + nrow * (int)blockIdx.y;   // this CTA's 32 (R = 4) or 16 streams
    {
      // 32 x 195 inputs, 13 per thread (idx = tid + 512 u): all global loads in flight together, then the stores
      float v[13];
#pragma unroll
      for (int u = 0; u < 13; u++) {
        const int idx = tid + u * 32 * P_EPI_WARPS, sl = idx & 31, j = idx >> 5, row = r0 + sl;
        v[u] = 0.f;
        if (idx < 32 * NET_C1_IN && sl < nrow && row < S)
          v[u] = j < 2 * NB_FEAT ? p.conv1_state[(size_t)row * 2 * NB_FEAT + j] : p.features[(size_t)row * NB_FEAT + j - 2 * NB_FEAT];
      }
#pragma unroll
      for (int u = 0; u < 13; u++) {
        const int idx = tid + u * 32 * P_EPI_WARPS;
        if (idx < 32 * NET_C1_IN) tmpT[idx] = v[u];
      }
    }
    // the words of the operand rows that the memory update moves down (read everything before anything is written)
    uint32_t rot[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int idx = tid + k * 32 * P_EPI_WARPS, sl = idx / (2 * W), w = idx - sl * 2 * W, row = r0 + sl;
      rot[k] = (sl < nrow && row < S) ? ((const uint32_t *)(p.c2in + (size_t)row * Kc))[W + w] : 0u;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * P_EPI_WARPS) : "memory");
    const int o = tid & 127, sg = tid >> 7;          // output, group of 8 streams
    if (o < cond && sg * 8 < nrow) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; i++) acc[i] = 0.f;
      const float *wp = p.conv1_w + o;
      // sequential FMA chain over the 195 inputs (sgemv order); the weights come from L2 / L1 in blocks of 13
      // independent loads, the next block requested before the current one is consumed (195 = 15 x 13)
      float wn[13];
#pragma unroll
      for (int u = 0; u < 13; u++) wn[u] = __ldg(wp + (size_t)u * cond);
      for (int j0 = 0; j0 < NET_C1_IN; j0 += 13) {
        float wc[13];
#pragma unroll
        for (int u = 0; u < 13; u++) wc[u] = wn[u];
        if (j0 + 13 < NET_C1_IN) {
#pragma unroll
          for (int u = 0; u < 13; u++) wn[u] = __ldg(wp + (size_t)(j0 + 13 + u) * cond);
        }
#pragma unroll
        for (int u = 0; u < 13; u++) {
          const int j = j0 + u;
          const float w = wc[u];
          const float4 a = *(const float4 *)&tmpT[j * 32 + sg * 8], b = *(const float4 *)&tmpT[j * 32 + sg * 8 + 4];
          acc[0] = fmaf(w, a.x, acc[0]); acc[1] = fmaf(w, a.y, acc[1]); acc[2] = fmaf(w, a.z, acc[2]); acc[3] = fmaf(w, a.w, acc[3]);
          acc[4] = fmaf(w, b.x, acc[4]); acc[5] = fmaf(w, b.y, acc[5]); acc[6] = fmaf(w, b.z, acc[6]); acc[7] = fmaf(w, b.w, acc[7]);
        }
      }
      const float bias = p.conv1_b[o];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int row = r0 + sg * 8 + i;
        if (row < S && !silence[row]) p.c2in[(size_t)row * Kc + 2 * cond + o] = (uint8_t)quant_u8(act_tanh(acc[i] + bias));
      }
    }
    // memory updates; silent frames leave both memories untouched (denoise.c:474)
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int idx = tid + k * 32 * P_EPI_WARPS, sl = idx / (2 * W), w = idx - sl * 2 * W, row = r0 + sl;
      if (sl < nrow && row < S && !silence[row]) ((uint32_t *)(p.c2in + (size_t)row * Kc))[w] = rot[k];
    }
    for (int idx = tid; idx < 32 * 2 * NB_FEAT; idx += 32 * P_EPI_WARPS) {
      const int sl = idx / (2 * NB_FEAT), j = idx - sl * 2 * NB_FEAT, row = r0 + sl;
      if (sl < nrow && row < S && !silence[row]) p.conv1_state[(size_t)row * 2 * NB_FEAT + j] = tmpT[(NB_FEAT + j) * 32 + sl];
    }
    fence_proxy_async();   // the operand rows are read back by TMA after the cluster barrier
  }

  const int njobs = NET_LAYERS * nslice;
  if (warp == P_EPI_WARPS) {
    // ------------------------------------------------------------------------------------------------
    // producer: lane 0 works, the whole warp takes part in the cluster barriers
    // ------------------------------------------------------------------------------------------------
    auto load_B = [&](int j) {
      const int L = j / nslice, s = j - L * nslice, st = ring_stage(j, P_STAGES);
      uint8_t *dst = sB + st * stage_bytes;
      if (L == 0) {
        const int batom = P_SLICE * TC_KATOM;
        mbar_expect_tx(bar_bfull(st), (uint32_t)(atoms_c * batom));
        for (int a = 0; a < atoms_c; a++)
          tma_load_2d(smem_u32(dst + a * batom), &maps.wi[0], bar_bfull(st), a * TC_KATOM, jq + s * P_SLICE);
      } else {
        const int batom = 3 * P_SLICE * TC_KATOM, row = (blockIdx.y * nslice + s) * 3 * P_SLICE;
        mbar_expect_tx(bar_bfull(st), (uint32_t)(2 * atoms_n * batom));
        for (int a = 0; a < atoms_n; a++) {
          tma_load_2d(smem_u32(dst + a * batom), &maps.wi[L], bar_bfull(st), a * TC_KATOM, row);
          tma_load_2d(smem_u32(dst + (atoms_n + a) * batom), &maps.wr[L], bar_bfull(st), a * TC_KATOM, row);
        }
      }
    };
    int fed = 0;   // jobs whose weights have been requested
    if (lane == 0) {
      // weights and GRU1's recurrent operand (previous frame's state) do not depend on conv1: fetched beside it
      for (; fed < P_STAGES && fed < njobs; fed++) load_B(fed);
      mbar_expect_tx(bar_h, (uint32_t)(atoms_n * TC_A_ATOM_BYTES));
      for (int a = 0; a < atoms_n; a++) tma_load_2d(smem_u32(sAh + a * TC_A_ATOM_BYTES), &maps.h[1], bar_h, a * TC_KATOM, m0);
    }
    __syncwarp();
    cluster_sync_all();   // every CTA is up (barriers initialised) and the conv1 prologues of the whole tile are in global memory
    if (lane == 0) {
      fence_proxy_async();
      mbar_expect_tx(bar_x, (uint32_t)(atoms_c * TC_A_ATOM_BYTES));
      for (int a = 0; a < atoms_c; a++) tma_load_2d(smem_u32(sAx + a * TC_A_ATOM_BYTES), &maps.x[0], bar_x, a * TC_KATOM, m0);
    }
    for (int L = 0; L < NET_LAYERS; L++) {
      if (lane == 0) {
        // the ring runs on into the next layer: job j reuses the stage of job j - P_STAGES (same pair, see ring_stage),
        // which belongs to this layer or an earlier one, so these waits never depend on the cluster barrier below
        const int until = (L + 1) * nslice + P_STAGES < njobs ? (L + 1) * nslice + P_STAGES : njobs;
        for (; fed < until; fed++) {
          mbar_wait(bar_bempty(ring_stage(fed, P_STAGES)), (uint32_t)((ring_use(fed, P_STAGES) - 1) & 1));
          load_B(fed);
        }
        if (L + 1 >= 2 && L + 1 < NET_LAYERS) {
          // the activation tiles are reusable once this layer's MMAs have retired: fetch the next layer's recurrent
          // operand right away (it only depends on the previous frame; GRU1's was loaded in the prologue)
          mbar_wait(bar_adone, (uint32_t)(L & 1));
          mbar_expect_tx(bar_h, (uint32_t)(atoms_n * TC_A_ATOM_BYTES));
          for (int a = 0; a < atoms_n; a++) tma_load_2d(smem_u32(sAh + a * TC_A_ATOM_BYTES), &maps.h[L + 1], bar_h, a * TC_KATOM, m0);
        }
      }
      if (L + 1 < NET_LAYERS) {
        __syncwarp();
        cluster_sync_all();   // all unit shares of layer L are in global memory
        if (lane == 0) {
          fence_proxy_async();
          mbar_expect_tx(bar_x, (uint32_t)(atoms_n * TC_A_ATOM_BYTES));
          for (int a = 0; a < atoms_n; a++) tma_load_2d(smem_u32(sAx + a * TC_A_ATOM_BYTES), &maps.x[L + 1], bar_x, a * TC_KATOM, m0);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------------------------------------
    // MMA + epilogue warpgroups
    // ------------------------------------------------------------------------------------------------
    cluster_sync_all();   // (pairs with the producer warp's: conv1 of the whole tile is published)
    const int pair = warp / P_PAIR_WARPS, mh = (warp >> 2) & 1;
    const int r0 = m0 + 64 * mh + frag_row(warp);
    bool live[2], silent[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      live[h] = r0 + 8 * h < S;
      silent[h] = live[h] ? silence[r0 + 8 * h] != 0 : true;
    }
    const uint32_t aX = smem_u32(sAx) + mh * TC_HALF_BYTES, aH = smem_u32(sAh) + mh * TC_HALF_BYTES;
    for (int L = 0; L < NET_LAYERS; L++) {
      const float *h_old = p.h_old[L];
      float *out_f32 = p.out_f32[L];
      uint8_t *out_u8 = p.out_u8[L];
      const float *pl = prm + (L == 0 ? 0 : 2 * upc + (L - 1) * 16 * upc);
      const int natoms = L == 0 ? atoms_c : atoms_n;
      mbar_wait(bar_x, (uint32_t)(L & 1));
      if (L >= 1) mbar_wait(bar_h, (uint32_t)((L - 1) & 1));
      const int j0 = L * nslice;
      for (int j = j0 + ((pair - j0) & 1); j < j0 + nslice; j += 2) {
        const int st = ring_stage(j, P_STAGES), ub = (j - j0) * P_SLICE;   // ub: first unit of the slice inside this CTA's share
        const uint32_t Bs = smem_u32(sB + st * stage_bytes);
        float outv[2][P_UPT];
        if (L > 0) {
          float hold[2][P_UPT];
#pragma unroll
          for (int h = 0; h < 2; h++) {   // old state: in flight while the MMAs run
            if (live[h]) frag_load_row(h_old + (size_t)(r0 + 8 * h) * N + jq + ub, hold[h]);
            else
#pragma unroll
              for (int q = 0; q < P_UPT; q++) hold[h][q] = 0.f;
          }
          int ai[3 * P_SLICE / 2], ar[3 * P_SLICE / 2];
#pragma unroll
          for (int i = 0; i < 3 * P_SLICE / 2; i++) ai[i] = ar[i] = 0;
          mbar_wait(bar_bfull(st), (uint32_t)(ring_use(j, P_STAGES) & 1));
          wgmma_fence();
          wgmma_chain_rt(ai, aX, TC_A_ATOM_BYTES, Bs, 3 * P_SLICE * TC_KATOM, natoms);
          wgmma_chain_rt(ar, aH, TC_A_ATOM_BYTES, Bs + natoms * 3 * P_SLICE * TC_KATOM, 3 * P_SLICE * TC_KATOM, natoms);
          wgmma_commit();
          wgmma_wait_all();
          wgmma_hold(ai); wgmma_hold(ar);
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_bempty(st));
#pragma unroll
          for (int h = 0; h < 2; h++) {
            if (silent[h]) {
#pragma unroll
              for (int q = 0; q < P_UPT; q++) outv[h][q] = hold[h][q];
            } else {
              gru_frag<P_SLICE>(ai, ar, pl + 16 * ub, h, hold[h], outv[h]);
            }
          }
        } else {
          int acc[P_SLICE / 2];
#pragma unroll
          for (int i = 0; i < P_SLICE / 2; i++) acc[i] = 0;
          mbar_wait(bar_bfull(st), (uint32_t)(ring_use(j, P_STAGES) & 1));
          wgmma_fence();
          wgmma_chain_rt(acc, aX, TC_A_ATOM_BYTES, Bs, P_SLICE * TC_KATOM, natoms);
          wgmma_commit();
          wgmma_wait_all();
          wgmma_hold(acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_bempty(st));
#pragma unroll
          for (int h = 0; h < 2; h++) conv_frag(acc, pl + ub, pl + upc + ub, h, outv[h]);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const size_t row = (size_t)(r0 + 8 * h);
          if (live[h]) frag_store_row(out_f32 + row * N + jq + ub, out_u8 + row * Kn + jq + ub, outv[h]);
        }
      }
      if (L + 1 < NET_LAYERS) {
        // this warp has finished reading the activation tiles of layer L
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_adone);
        // this thread's part of layer L is written: make it visible to the TMA (async proxy) reads of the whole
        // cluster, then wait until every CTA has done the same
        fence_proxy_async();
        cluster_sync_all();
      }
    }
  }
  cluster_sync_all();   // no CTA of the cluster exits while a peer could still be arriving on the cluster barrier
}
