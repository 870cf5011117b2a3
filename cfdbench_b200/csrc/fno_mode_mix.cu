// K2 -- per-mode complex channel mix on the tensor cores:  Y[k][b][o] = sum_i X[k][b][i] * Wk[k][i][o].
//
// Replaces the two torch.einsum("bixy,ioxy->boxy") corner products plus the zero-filled
// (B,32,64,33) cfloat buffer of the reference (src/models/fno/fno2d.py:54-57, 65-78).
//
// Modes are stored mode-major (xm[k][b][c], written that way by the forward DFT kernels), so the 128 rows of a tile are
// one contiguous 32 KB block.  For one mode k the mix over a tile of 128 samples is a real GEMM on the interleaved
// complex64 rows exactly as they sit in memory:
//     D[128 samples][64 = (o, re|im)] = A[128][64 = (i, re|im)] * B_k^T         (wgmma m64n64k8 tf32, K = 64)
//     B_k[(o,re)][(i,re)] = Wre,  B_k[(o,re)][(i,im)] = -Wim,  B_k[(o,im)][(i,re)] = Wim,  B_k[(o,im)][(i,im)] = Wre
// run as 3xTF32.  The B operand of every mode is prepared once per weight update (pack_mix_operand_*_kernel:
// real-expanded, split into tf32 hi/lo, laid out as the K-major operand image) and arrives with ONE 32 KB bulk copy per mode.
//
//   * work item = one MODE (all its sample tiles): B_k is fetched once per mode, 288 items on the persistent CTAs;
//   * warp 8 lane 0 -- producer: the A tile is the raw fp32 block itself, dropped by TMA (two {32 floats, 128 rows}
//     boxes, 128-byte swizzle) into a 4-slot ring.  At B = 256 (two tiles per mode, two or three modes per CTA) the
//     ring holds all or most of the tiles of a CTA, so nearly every load is in flight from the start;
//   * warpgroups 0 and 1 -- rows 0..63 / 64..127 of every tile: each thread reads its A fragments out of the swizzled
//     tile (conflict-free) and splits them into tf32 hi / lo in registers; then A_hi x B_hi, A_hi x B_lo, A_lo x B_hi
//     (24 register-A MMAs), after which the slot is released, and the epilogue from the accumulator registers: mode-major
//     ym rows (fp32 path / backward) or the per-sample operand image of block_fused_kernel's inverse-kx GEMM (tf32 hi/lo
//     split).
// With the conj-transposed pack the same kernel is the adjoint mix of the backward pass
// (Xbar[b,i,k] = sum_o G[b,o,k] conj(W[i,o,k]), SURVEY.md 8a).
#include "fno_common.cuh"
#include "tc_common.cuh"
#include "tc_tma.cuh"

namespace fno {

constexpr int kMxM = 128;        // samples per tile
constexpr int kMxK = 2 * kC;     // 64 real (i, re|im)
constexpr int kMxN = 2 * kC;     // 64 real (o, re|im)
constexpr uint32_t kMxLboB = (kMxN / 8) * 128;       // 1024
constexpr int kMxBFloats = kMxN * kMxK;              // 4096 per image (hi or lo)
constexpr int kMxOperandFloats = 2 * kMxBFloats;     // per mode: hi image then lo image (32 KB)
constexpr int kMxConsumerWarps = 8;
constexpr int kMxProdWarp = 8;
constexpr int kMxThreads = 9 * 32;
constexpr int kMxRing = 4;                           // A slots
constexpr uint32_t kMxABytes = kMxM * kMxK * 4;      // 32,768 B per tile: two K halves of 128 rows x 128 B
constexpr uint32_t kMxBBytes = kMxOperandFloats * 4; // 32,768 B per mode
constexpr size_t kMxImageBytes = 147456;             // per sample: [hi|lo][ky 12][48 rows][32 o] fp32
constexpr int kMxStageLd = kMxN + 1;                 // padded row of the staged result tile

struct MxSmem {
  alignas(1024) unsigned char a[kMxRing][kMxABytes];   // raw fp32 tiles (TMA, 128B swizzle)
  alignas(1024) float b[2][kMxOperandFloats];          // [mode parity] hi | lo images
  float stage[2][64 * kMxStageLd];                      // per warpgroup: its 64 x 64 result tile (image epilogue)
  alignas(8) uint64_t a_full[kMxRing], a_free[kMxRing];
  uint64_t b_full[2], b_free[2];
};

__global__ void __launch_bounds__(kMxThreads, 1)
    mode_mix_tc_kernel(const __grid_constant__ CUtensorMap x_map, const float* __restrict__ wop, float2* __restrict__ ym,
                       unsigned char* __restrict__ ym_img, int batch, int n_btiles) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  MxSmem& sm = *reinterpret_cast<MxSmem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
  const int tid = threadIdx.x, lane = tid & 31, warp = tc::warp_index_uniform();

  // modes of this CTA: k = first + j * stride; tiles are numbered t = j * n_btiles + bt in processing order
  const int first = blockIdx.x, stride = gridDim.x;
  const int n_modes = (first < kModes) ? (kModes - first + stride - 1) / stride : 0;

  if (tid == 0) {
    for (int i = 0; i < kMxRing; ++i) {
      mbar_init(&sm.a_full[i], 1);
      mbar_init(&sm.a_free[i], kMxConsumerWarps);
    }
    for (int i = 0; i < 2; ++i) { mbar_init(&sm.b_full[i], 1); mbar_init(&sm.b_free[i], kMxConsumerWarps); }
    fence_mbar_init();
    // the weights of the first two modes do not depend on the previous kernel of the chain: fetch them now
    for (int j = 0; j < 2 && j < n_modes; ++j) {
      mbar_expect_tx(&sm.b_full[j], kMxBBytes);
      bulk_g2s(sm.b[j], wop + static_cast<size_t>(first + j * stride) * kMxOperandFloats, kMxBBytes, &sm.b_full[j]);
    }
  }
  __syncthreads();
  pdl_wait();  // xm comes from the previous kernel of the chain
  pdl_launch_dependents();

  if (warp < kMxConsumerWarps) {
    const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
    const int m0 = 64 * wg + 16 * wq + (lane >> 2);   // fragment rows m0, m0 + 8 of the tile
    int t = 0;
#pragma unroll 1
    for (int j = 0; j < n_modes; ++j) {
      const int k = first + j * stride;
      mbar_wait(&sm.b_full[j & 1], (j >> 1) & 1);
      const uint32_t b_hi = tc::smem_addr(sm.b[j & 1]), b_lo = b_hi + kMxBFloats * 4;
#pragma unroll 1
      for (int bt = 0; bt < n_btiles; ++bt, ++t) {
        const int s = t % kMxRing;
        mbar_wait(&sm.a_full[s], (t / kMxRing) & 1);
        // A fragments: element (m, k) of the tile sits in K half k / 32, line m, 16-byte chunk ((k % 32) / 4) ^ (m & 7)
        uint32_t a_hi[8][4], a_lo[8][4];
#pragma unroll
        for (int ks = 0; ks < kMxK / 8; ++ks)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int m = m0 + 8 * (r & 1), chunk = 2 * (ks & 3) + (r >> 1);
            const float x = *reinterpret_cast<const float*>(sm.a[s] + (ks >> 2) * (kMxABytes / 2) + m * 128 +
                                                            ((chunk ^ (m & 7)) << 4) + q * 4);
            float hi, lo;
            tc::split_tf32(x, hi, lo);
            a_hi[ks][r] = __float_as_uint(hi);
            a_lo[ks][r] = __float_as_uint(lo);
          }
        float acc[32];
        tc::wg_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {   // A_hi x B_hi, A_hi x B_lo, A_lo x B_hi
          const uint32_t pb = pass == 1 ? b_lo : b_hi;
#pragma unroll
          for (int ks = 0; ks < kMxK / 8; ++ks)
            tc::wg_tf32_rs_n64(acc, pass == 2 ? a_lo[ks] : a_hi[ks], tc::make_smem_desc(pb + ks * 2 * kMxLboB, kMxLboB, 128),
                               (pass | ks) ? 1u : 0u);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc(acc);
        // the MMAs have consumed the fragments loaded from the A slot (and, after the last tile of the mode, the B slot):
        // the producer may refill them
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&sm.a_free[s]);
          if (bt == n_btiles - 1) mbar_arrive(&sm.b_free[j & 1]);
        }
        // acc[4 i + 2 hh + e] = D[m0 + 8 hh][8 i + 2 q + e]: output channel o = 4 i + q, e = re | im
        if (ym_img == nullptr) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int b = bt * kMxM + m0 + 8 * hh;
            if (b >= batch) continue;
            float2* dst = ym + (static_cast<size_t>(k) * batch + b) * kC + q;
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[4 * i] = make_float2(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
          }
        } else {
          // Operand image of block_fused_kernel's inverse-kx GEMM (fno_block_fused.cu): per sample
          // [hi|lo][ky][48 rows][32 o] fp32, row = 24 (kxi & 1) + 2 (kxi >> 1) + (re|im), 32-byte chunks XOR-swizzled
          // with (row & 3); tf32 hi / lo split here so the consumer only copies and multiplies.  A sample's (re|im) row of
          // this mode is one 128-byte line: the tile goes through shared memory so that a warp stores whole lines
          // (lane = o).
          float* stg = sm.stage[wg];
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              stg[(m0 - 64 * wg + 8 * hh) * kMxStageLd + 8 * i + 2 * q] = acc[4 * i + 2 * hh];
              stg[(m0 - 64 * wg + 8 * hh) * kMxStageLd + 8 * i + 2 * q + 1] = acc[4 * i + 2 * hh + 1];
            }
          tc::named_barrier(1 + wg, 128);
          const int kxi = k / kM2, ky = k % kM2;
#pragma unroll 4
          for (int rr = 0; rr < 16; ++rr) {
            const int r = 16 * wq + rr, b = bt * kMxM + 64 * wg + r;
            if (b >= batch) break;
            unsigned char* img = ym_img + static_cast<size_t>(b) * kMxImageBytes + ky * 6144;
#pragma unroll
            for (int ri = 0; ri < 2; ++ri) {
              const int row = 24 * (kxi & 1) + 2 * (kxi >> 1) + ri;
              float hi, lo;
              tc::split_tf32(stg[r * kMxStageLd + 2 * lane + ri], hi, lo);
              unsigned char* dst = img + row * 128 + (((lane >> 3) ^ (row & 3)) << 5) + (lane & 7) * 4;
              *reinterpret_cast<float*>(dst) = hi;
              *reinterpret_cast<float*>(dst + kMxImageBytes / 2) = lo;
            }
          }
          tc::named_barrier(1 + wg, 128);   // the tile buffer is free for the next tile
        }
      }
    }
  } else if (warp == kMxProdWarp && lane == 0) {
    int t = 0;
    for (int j = 0; j < n_modes; ++j) {
      const int k = first + j * stride;
      if (j >= 2) {   // modes 0 and 1 were requested in the prologue
        mbar_wait(&sm.b_free[j & 1], ((j >> 1) - 1) & 1);
        mbar_expect_tx(&sm.b_full[j & 1], kMxBBytes);
        bulk_g2s(sm.b[j & 1], wop + static_cast<size_t>(k) * kMxOperandFloats, kMxBBytes, &sm.b_full[j & 1]);
      }
      for (int bt = 0; bt < n_btiles; ++bt, ++t) {
        const int s = t % kMxRing;
        if (t >= kMxRing) mbar_wait(&sm.a_free[s], ((t / kMxRing) - 1) & 1);
        mbar_expect_tx(&sm.a_full[s], kMxABytes);
        const int row0 = k * batch + bt * kMxM;   // rows past this mode's samples are never stored by the epilogue
        tma_load_2d(sm.a[s], &x_map, 0, row0, &sm.a_full[s]);
        tma_load_2d(sm.a[s] + kMxABytes / 2, &x_map, 32, row0, &sm.a_full[s]);
      }
    }
  }
}

size_t ym_image_bytes(int batch) { return static_cast<size_t>(batch) * kMxImageBytes; }

// ym_img != nullptr: write the per-sample inverse-kx operand image (see the epilogue) instead of the mode-major ym.
cudaError_t launch_mode_mix(const void* xm, const void* wop, void* ym, void* ym_img, int batch, cudaStream_t stream) {
  auto kern = mode_mix_tc_kernel;
  constexpr size_t smem = sizeof(MxSmem);
  static PerDeviceLaunch pd;
  int n_sm = 0;
  cudaError_t e0 = per_device_setup(kern, smem, pd, &n_sm);
  if (e0 != cudaSuccess) return e0;
  if (reinterpret_cast<uintptr_t>(xm) & 15) return cudaErrorMisalignedAddress;
  // the mode-major spectrum as rows of 64 floats: [288 * batch rows][64], box {32 floats, 128 rows}
  CUtensorMap map;
  e0 = make_tma_map_2d(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, xm, kMxK, static_cast<uint64_t>(kModes) * batch, 32, kMxM);
  if (e0 != cudaSuccess) return e0;
  const int n_btiles = (batch + kMxM - 1) / kMxM;
  const int grid = kModes < n_sm ? kModes : n_sm;
  return launch_chained(kern, dim3(grid), dim3(kMxThreads), smem, stream, map, static_cast<const float*>(wop),
                        static_cast<float2*>(ym), static_cast<unsigned char*>(ym_img), batch, n_btiles);
}

// ------------------------------------------------------------------------------------------------
// B operand image of the mix, built from the packed weights Wk[k][i][o] (pack_spectral_kernel below):
// per mode 2 x 4096 floats (tf32 hi image, then lo image), element (n = 2o + part, kk = 2i + ri) at
// tc::kmajor_offset(n, kk, 64).
// ------------------------------------------------------------------------------------------------
__global__ void pack_mix_operand_kernel(const float2* __restrict__ wk, float* __restrict__ wop) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // over k*1024 + i*32 + o
  if (idx >= kModes * kC * kC) return;
  const int k = idx / (kC * kC), i = (idx / kC) % kC, o = idx % kC;
  const float2 w = wk[idx];
  float* img = wop + static_cast<size_t>(k) * kMxOperandFloats;
  const float val[2][2] = {{w.x, -w.y}, {w.y, w.x}};  // [part of the output][re|im of the input]
#pragma unroll
  for (int part = 0; part < 2; ++part)
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      float hi, lo;
      tc::split_tf32(val[part][ri], hi, lo);
      const uint32_t off = tc::kmajor_offset(2 * o + part, 2 * i + ri, kMxN) / 4;
      img[off] = hi;
      img[kMxBFloats + off] = lo;
    }
}

cudaError_t launch_pack_mix_operand(const void* wk, void* wop, cudaStream_t stream) {
  const int n = kModes * kC * kC;
  pack_mix_operand_kernel<<<(n + 255) / 256, 256, 0, stream>>>(static_cast<const float2*>(wk), static_cast<float*>(wop));
  return cudaGetLastError();
}

size_t mix_operand_bytes() { return static_cast<size_t>(kModes) * kMxOperandFloats * sizeof(float); }

// The same image straight from the reference parameter layout (weights1/2: (Cin, Cout, 12, 12) complex64), one
// launch per layer and direction: a thread produces one 16-byte operand chunk (row n, 4 consecutive kk) of both the
// hi and the lo image, so the writes are coalesced; the 2.36 MB of weights are gathered through L2.  This is what
// runs after every optimizer step.
__global__ void pack_mix_operand_direct_kernel(const float2* __restrict__ w1, const float2* __restrict__ w2,
                                               float* __restrict__ wop, int conj_transpose) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // over k * 1024 + (kk/4) * 64 + n: the operand's own order
  if (idx >= kModes * 1024) return;
  const int k = idx >> 10, kq = (idx >> 6) & 15, n = idx & 63;
  const int kxi = k / kM2, ky = k % kM2;
  const float2* src = (kxi < kM1) ? w1 : w2;
  const int kk_mode = (kxi % kM1) * kM2 + ky;
  const int a = n >> 1, part = n & 1;  // output channel (o) of the mix and its re|im
  float v[4];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int c = 2 * kq + j;  // input channel (i) of the mix
    // forward: Wk[k][i = c][o = a] = W[c][a][k];  adjoint: Wk[k][i = c][o = a] = conj(W[a][c][k])
    const int wi = conj_transpose ? a : c, wo = conj_transpose ? c : a;
    float2 w = __ldg(src + (static_cast<size_t>(wi) * kC + wo) * (kM1 * kM2) + kk_mode);
    if (conj_transpose) w.y = -w.y;
    v[2 * j + 0] = part ? w.y : w.x;    // (o,re): [Wre, -Wim]   (o,im): [Wim, Wre]
    v[2 * j + 1] = part ? w.x : -w.y;
  }
  float4 hi, lo;
  tc::split_tf32(v[0], hi.x, lo.x);
  tc::split_tf32(v[1], hi.y, lo.y);
  tc::split_tf32(v[2], hi.z, lo.z);
  tc::split_tf32(v[3], hi.w, lo.w);
  float* img = wop + static_cast<size_t>(k) * kMxOperandFloats;
  const uint32_t off = tc::kmajor_offset(n, 4 * kq, kMxN) / 4;
  *reinterpret_cast<float4*>(img + off) = hi;
  *reinterpret_cast<float4*>(img + kMxBFloats + off) = lo;
}

cudaError_t launch_pack_mix_operand_direct(const void* w1, const void* w2, void* wop, int conj_transpose,
                                           cudaStream_t stream) {
  const int n = kModes * 1024;
  pack_mix_operand_direct_kernel<<<(n + 255) / 256, 256, 0, stream>>>(
      static_cast<const float2*>(w1), static_cast<const float2*>(w2), static_cast<float*>(wop), conj_transpose);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Weight packing: reference parameter layout (Cin, Cout, 12, 12) complex64 x2 (weights1, weights2;
// reference fno2d.py:31-51)  ->  Wk[k][i][o], k = kxi*12 + ky, kxi<12 from weights1 else weights2.
// conj_transpose=1 writes Wk[k][o][i] = conj(W[i][o][k]) (the operand of the adjoint mix:
// Xbar[b,i,k] = sum_o G[b,o,k] conj(W[i,o,k]), SURVEY.md 8a).
// ------------------------------------------------------------------------------------------------
__global__ void pack_spectral_kernel(const float2* __restrict__ w1, const float2* __restrict__ w2,
                                     float2* __restrict__ wk, int conj_transpose) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // over k*1024 + a*32 + c
  if (idx >= kModes * kC * kC) return;
  const int k = idx / (kC * kC);
  const int a = (idx / kC) % kC, c = idx % kC;
  const int i = conj_transpose ? c : a;
  const int o = conj_transpose ? a : c;
  const int kxi = k / kM2, ky = k % kM2;
  const float2* src = (kxi < kM1) ? w1 : w2;
  const int kk = (kxi % kM1) * kM2 + ky;
  float2 v = src[(static_cast<size_t>(i) * kC + o) * (kM1 * kM2) + kk];
  if (conj_transpose) v.y = -v.y;
  wk[idx] = v;
}

cudaError_t launch_pack_spectral(const void* w1, const void* w2, void* wk, int conj_transpose, cudaStream_t stream) {
  const int n = kModes * kC * kC;
  pack_spectral_kernel<<<(n + 255) / 256, 256, 0, stream>>>(static_cast<const float2*>(w1), static_cast<const float2*>(w2),
                                                           static_cast<float2*>(wk), conj_transpose);
  return cudaGetLastError();
}

// inverse of the pack for gradients: gWk[k][i][o] -> gw1/gw2 (Cin, Cout, 12, 12).  kAccum: add to gw1/gw2 instead of
// overwriting them (the rollout backward sums the steps of its sweep into one gradient)
template <bool kAccum>
__global__ void unpack_spectral_kernel(const float2* __restrict__ gwk, float2* __restrict__ gw1,
                                       float2* __restrict__ gw2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // over (i*32+o)*144 + kk for both halves
  if (idx >= 2 * kC * kC * kM1 * kM2) return;
  const int half = idx / (kC * kC * kM1 * kM2);
  const int r = idx % (kC * kC * kM1 * kM2);
  const int io = r / (kM1 * kM2), kk = r % (kM1 * kM2);
  const int k = (half * kM1 + kk / kM2) * kM2 + kk % kM2;
  const float2 v = gwk[static_cast<size_t>(k) * kC * kC + io];
  float2* dst = (half ? gw2 : gw1) + r;
  if constexpr (kAccum) {
    const float2 o = *dst;
    *dst = make_float2(o.x + v.x, o.y + v.y);
  } else {
    *dst = v;
  }
}

cudaError_t launch_unpack_spectral(const void* gwk, void* gw1, void* gw2, int accumulate, cudaStream_t stream) {
  const int n = 2 * kC * kC * kM1 * kM2;
  auto kern = accumulate ? unpack_spectral_kernel<true> : unpack_spectral_kernel<false>;
  kern<<<(n + 255) / 256, 256, 0, stream>>>(static_cast<const float2*>(gwk), static_cast<float2*>(gw1),
                                            static_cast<float2*>(gw2));
  return cudaGetLastError();
}

}  // namespace fno
