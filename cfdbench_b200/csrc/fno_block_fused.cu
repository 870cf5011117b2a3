// Fused Fourier-block output stage for bf16 activation storage (inference):
//   out[b][o][h][w] = GELU( irfft2(pad(Y))[b][o][h][w] + sum_i W0[o][i] x[b][i][h][w] + bias[o] )       (bf16 in, bf16 out)
// replacing irfft2 + Conv2d(32,32,1) + add + GELU of the reference FnoBlock (src/models/fno/fno2d.py:65-72,81,104-111)
// with one kernel in which the half-inverted spectrum Z never leaves the SM.
//
// Work unit = (sample, chunk of 16 image rows); a CTA always works on the same chunk (blockIdx.x % 4), so its inverse-kx
// constant is loaded once.  Per unit:
//   GEMM1 (inverse DFT along kx, 3xTF32):  Z1[(ky, o) 384][(h', re|im) 32] = Y^T[(ky, o)][(kx, re|im) 48] * F[(h', ri)][.]^T
//          six m64n32k8 chains, one per ky pair; A = the mode image of the sample (fno_mode_mix.cu writes it with the
//          tf32 hi/lo split done), loaded from the warpgroup's image slot into A-fragment registers -- the image's
//          32-byte chunk swizzle makes those loads conflict-free -- and B = the constant F (K-major); Z1 -> tf32 hi/lo ->
//          Zt, the K-major B operand of GEMM2 per image row (96 KB for 16 rows).  GEMM1's M rows are ordered so that a thread's two fragment rows are
//          the two ky of its pair at one channel: its four values of an (h', o) form one 16-byte chunk of Zt, one
//          st.shared.v4 per hi / lo.  Bias rides in the row that irfft2's C2R stage ignores (Im of ky = 0).
//   GEMM2 per image row h:  D[64 w][32 o] = E[w][(ky, ri) 24] Zt_h + X_h[w][32 i] W0^T
//          E Zt_h: m64n32k8 tf32, 3xTF32 (E = C2R stage with c_ky/HW folded in, fno_block_tc.cu builds it); E's hi / lo
//          A fragments are loaded into registers once per CTA, so only Zt_h is read from shared memory.
//          X_h W0^T: m64n32k16 bf16, A = the row of the TMA slot that holds it as [i][w], read once per row by
//          ldmatrix.trans into A fragments and used by all three bf16 terms of W0 (24 mantissa bits), accumulated into
//          the same fp32 registers.  x is exact in bf16.
//          Epilogue exact-erf GELU -> bf16x2 -> stmatrix.trans into the swizzled [o][w] staging tile -> one TMA store
//          per row.
// Roles: warpgroups 0 / 1 -- the even / odd ky pairs of GEMM1 and the even / odd rows of GEMM2.  Each warpgroup owns
// one image slot (24 KB = one ky pair, hi + lo, two bulk copies by its thread 0) and reads the three pairs of the next
// unit from it into three fragment sets during GEMM2, one pair every other row; the slot is refilled right after the
// row barrier that follows its reads.  So GEMM1 waits for no image, and with two accumulator sets pair 1's MMAs run
// while pair 0 is split and stored, pair 2's while pair 1 is.  (A ninth, producer warp would cap the registers at
// those of three warpgroups, 168, too few for the fragment sets.)  Each warpgroup owns a ring of kFzXSlots activation
// rows; its thread 0 refills a slot as soon as the MMAs that read it have completed, so the ring runs up to kFzXSlots rows
// ahead, across GEMM1 and across unit boundaries.  GEMM2 keeps two accumulator sets: the MMAs of row r + 1 run while row
// r's epilogue does.
#include "fno_common.cuh"
#include "tc_common.cuh"
#include "tc_tma.cuh"
#include <math.h>
#include <string.h>

namespace fno {

constexpr int kFzRows = 16;                            // image rows per unit
constexpr int kFzChunks = kH / kFzRows;                // 4
constexpr int kFzWgRows = kFzRows / 2;                 // GEMM2 rows per warpgroup and unit
constexpr int kFzThreads = 8 * 32;                     // 2 warpgroups
constexpr int kZK = 2 * kM2;                           // 24: (ky, re|im)
constexpr int kImgK = 2 * kKX;                         // 48: (kx, re|im) image rows
constexpr size_t kYmImgBytes = 147456;                 // per sample: [hi|lo][ky 12][48 rows][32 o] fp32
constexpr uint32_t kImgKyBytes = kImgK * kC * 4;       // 6144: one ky of the hi or the lo image
constexpr uint32_t kFzStage = 4 * kImgKyBytes;         // one ky pair: hi (2 x 6144 B) then lo
constexpr int kFzFFloats = 2 * (2 * kFzRows) * kImgK;  // [n = 2 h' + ri (32)][48], hi | lo: per chunk
constexpr int kFzEFloats = 2 * kW * kZK;               // [64 w][24] hi | lo
constexpr uint32_t kFzZtFloats = kC * kZK;             // one image row, hi or lo: [32 o][24 k] K-major
constexpr uint32_t kLboF = (2 * kFzRows / 8) * 128;    // 512
constexpr uint32_t kLboO = (kC / 8) * 128;             // 512: B operands with 32 rows (o)
// One image row of all 32 channels of a bf16 activation: TMA box {w 64, h 1, (b, c) 32}, [c][w] with the 128-byte swizzle.
// The same box is the load of x and the store of out.
constexpr uint32_t kFzBoxW = kW, kFzBoxH = 1, kFzBoxC = kC;
constexpr uint32_t kFzRowBytes = kFzBoxW * kFzBoxH * kFzBoxC * 2;   // 4096 = expect_tx of one fill
constexpr int kFzXSlots = 4;                                         // activation rows in flight per warpgroup
constexpr uint32_t kFzW0Bytes = kC * kC * 2;                         // one bf16 term of W0, K-major

// Activation ring of a warpgroup: fill n (n = kFzWgRows * unit + r, r-th GEMM2 row of the unit) goes to slot n % S and
// completes phase n / S of that slot's barrier.  The same two functions are used where a fill is issued and waited for.
__host__ __device__ constexpr int fz_x_slot(int n) { return n % kFzXSlots; }
__host__ __device__ constexpr uint32_t fz_x_parity(int n) { return static_cast<uint32_t>(n / kFzXSlots) & 1u; }

struct FzSmem {
  alignas(1024) unsigned char x[2][kFzXSlots][kFzRowBytes];   // per warpgroup: activation ring (TMA, 128B swizzle)
  alignas(1024) unsigned char st[2][2][kFzRowBytes];          // per warpgroup: double-buffered output staging tile
  alignas(128) unsigned char y[2][kFzStage];           // per warpgroup: image slot
  alignas(128) float zt[kFzRows][2][kFzZtFloats];      // GEMM2 B operand per row: hi, lo
  alignas(128) float f_hi[kFzFFloats / 2];
  alignas(128) float f_lo[kFzFFloats / 2];
  alignas(128) unsigned char w0[3][kFzW0Bytes];        // B[n = o][k = i] = W0[o][i] = t1 + t2 + t3 (bf16 terms)
  alignas(16) float bias[kC];
  alignas(8) uint64_t y_full[2];
  alignas(8) uint64_t x_full[2][kFzXSlots];
};
static_assert(sizeof(FzSmem) <= 232448, "block_fused_kernel: shared memory over the per-block opt-in limit");

// byte offset of (line, element e) in a 128-byte-swizzled image of 128-byte lines of bf16 (what TMA writes / reads)
__device__ __forceinline__ uint32_t sw128_bf16_offset(int line, int e) {
  return static_cast<uint32_t>(line * 128 + ((((e >> 3) ^ line) & 7) << 4) + (e & 7) * 2);
}

__global__ void __launch_bounds__(kFzThreads, 1)
    block_fused_kernel(const __grid_constant__ CUtensorMap x_map, const __grid_constant__ CUtensorMap out_map,
                       const unsigned char* __restrict__ img, const float* __restrict__ w0t,
                       const float* __restrict__ bias, const float* __restrict__ etab, const float* __restrict__ ftab,
                       int batch) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  FzSmem& sm = *reinterpret_cast<FzSmem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();   // the TMA swizzle atoms need 1024-byte alignment
  const int tid = threadIdx.x, lane = tid & 31, warp = tc::warp_index_uniform();
  const int chunk = blockIdx.x % kFzChunks, b0 = blockIdx.x / kFzChunks, bstride = gridDim.x / kFzChunks;
  const int n_units = b0 < batch ? (batch - b0 + bstride - 1) / bstride : 0;

  // ---------------------------------------------------------------- prologue (constants and weights only)
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&sm.y_full[i], 1);   // thread 0 of the warpgroup: expect_tx
      for (int s = 0; s < kFzXSlots; ++s) mbar_init(&sm.x_full[i][s], 1);   // thread 0 of the warpgroup: expect_tx
    }
    fence_mbar_init();
  }
  for (int e = tid; e < kFzFFloats / 2; e += kFzThreads) {
    sm.f_hi[e] = __ldg(ftab + chunk * kFzFFloats + e);
    sm.f_lo[e] = __ldg(ftab + chunk * kFzFFloats + kFzFFloats / 2 + e);
  }
  for (int e = tid; e < kC * kC; e += kFzThreads) {  // B[n = o][k = i] = W0[o][i] = w0t[i][o]: three bf16 terms
    const int i = e / kC, o = e % kC;
    const float w = w0t[e];
    const __nv_bfloat16 t1 = __float2bfloat16_rn(w);
    const float r1 = w - __bfloat162float(t1);
    const __nv_bfloat16 t2 = __float2bfloat16_rn(r1);
    const __nv_bfloat16 t3 = __float2bfloat16_rn(r1 - __bfloat162float(t2));
    const uint32_t off = static_cast<uint32_t>(((i >> 3) * (kC / 8) + (o >> 3)) * 128 + (o & 7) * 16 + (i & 7) * 2);
    *reinterpret_cast<__nv_bfloat16*>(sm.w0[0] + off) = t1;
    *reinterpret_cast<__nv_bfloat16*>(sm.w0[1] + off) = t2;
    *reinterpret_cast<__nv_bfloat16*>(sm.w0[2] + off) = t3;
  }
  if (tid < kC) sm.bias[tid] = bias != nullptr ? bias[tid] : 0.f;
  tc::fence_proxy_async_smem();   // the constant operands above are read by the tensor cores
  __syncthreads();
  pdl_wait();   // the image and x come from the previous kernels of the chain
  pdl_launch_dependents();

  const int g = warp >> 2, wq = warp & 3, q = lane & 3, t = tid & 127;
  const int m0 = 16 * wq + (lane >> 2);   // fragment rows m0, m0 + 8
  const int n_fills = kFzWgRows * n_units;
  // fill n of this warpgroup's activation ring: row h = 16 chunk + g + 2 r of unit u, all 32 channels (thread t == 0)
  auto x_fill = [&](int n) {
    const int u = n / kFzWgRows, r = n % kFzWgRows, s = fz_x_slot(n);
    mbar_expect_tx(&sm.x_full[g][s], kFzRowBytes);
    tma_load_3d(sm.x[g][s], &x_map, 0, kFzRows * chunk + g + 2 * r, (b0 + u * bstride) * kC, &sm.x_full[g][s]);
  };
  // fill f of this warpgroup's image slot: ky pair g + 2 (f % 3) of unit f / 3, hi and lo (thread t == 0); fill f
  // completes phase f of y_full[g] and is issued once all 128 threads have read fill f - 1
  const int n_yfills = 3 * n_units;
  auto y_fill = [&](int f) {
    const unsigned char* src = img + static_cast<size_t>(b0 + (f / 3) * bstride) * kYmImgBytes +
                               (g + 2 * (f % 3)) * (kFzStage / 2);
    mbar_expect_tx(&sm.y_full[g], kFzStage);
    bulk_g2s(sm.y[g], src, kFzStage / 2, &sm.y_full[g]);
    bulk_g2s(sm.y[g] + kFzStage / 2, src + kYmImgBytes / 2, kFzStage / 2, &sm.y_full[g]);
  };
  if (t == 0) {
    if (n_yfills > 0) y_fill(0);
    for (int n = 0; n < kFzXSlots && n < n_fills; ++n) x_fill(n);
  }
  const uint32_t w0_s = tc::smem_addr(sm.w0[0]);
  // A fragments of E (tf32 m64k8, rows w = m0, m0 + 8) for the C2R passes of every row: e_frag[0 / 1] = hi / lo
  uint32_t e_frag[2][kZK / 8][4];
#pragma unroll
  for (int hl = 0; hl < 2; ++hl)
#pragma unroll
    for (int ks = 0; ks < kZK / 8; ++ks)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t off = tc::kmajor_offset(m0 + 8 * (j & 1), 8 * ks + q + 4 * (j >> 1), kW) / 4;
        e_frag[hl][ks][j] = __float_as_uint(__ldg(etab + hl * (kFzEFloats / 2) + off));
      }

  // GEMM1 row m = 16 wq + 8 hh + j holds ky = 2p + hh and channel o = 8 wq + j, so the fragment rows m0, m0 + 8 of a
  // thread are (2p, o1) and (2p + 1, o1) with o1 = 8 wq + lane / 4.
  const int o1 = 8 * wq + (lane >> 2);
  // A fragments of fill f of the slot, tf32 hi [0] / lo [1]: A[m][kk] = image[2p + hh][kk][o], line kk of the ky,
  // 32-byte chunk (o / 8) ^ (kk & 3) = wq ^ (kk & 3), word o & 7; the lanes of a load cover 8 words of 4 chunks with
  // distinct swizzle phases: no bank conflicts.
  auto load_pair = [&](uint32_t (&a)[2][kImgK / 8][4], int f) {
    mbar_wait(&sm.y_full[g], f & 1);
#pragma unroll
    for (int ks = 0; ks < kImgK / 8; ++ks)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int kk = 8 * ks + q + 4 * (r >> 1);
        const uint32_t off = (r & 1) * kImgKyBytes + kk * 128 + ((wq ^ (kk & 3)) << 5) + (lane >> 2) * 4;
        a[0][ks][r] = *reinterpret_cast<const uint32_t*>(sm.y[g] + off);
        a[1][ks][r] = *reinterpret_cast<const uint32_t*>(sm.y[g] + kFzStage / 2 + off);
      }
  };
  // the 18 MMAs of one ky pair, one commit group: Y_hi F_hi + Y_lo F_hi + Y_hi F_lo
  auto issue_pair = [&](float (&acc)[16], const uint32_t (&a)[2][kImgK / 8][4]) {
    tc::wg_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      const uint32_t fb = tc::smem_addr(pass == 2 ? sm.f_lo : sm.f_hi);
#pragma unroll
      for (int ks = 0; ks < kImgK / 8; ++ks)
        tc::wg_tf32_rs_n32(acc, a[pass == 1][ks], tc::make_smem_desc(fb + ks * 2 * kLboF, kLboF, 128),
                           (pass | ks) ? 1u : 0u);
    }
    tc::wg_commit();
  };
  // acc[4 i + 2 hh + e] = Z1[(2p + hh, o1)][n = 8 i + 2 q + e]: row h' = 4 i + q, k = 4p + 2 hh + e, i.e. the four
  // values of a given i are the 16-byte chunk (o1, k = 4p .. 4p + 3) of Zt row h'
  auto store_pair = [&](const float (&acc)[16], int p) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v[4] = {acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]};
      if (p == 0) v[1] = sm.bias[o1];   // Im of ky = 0: C2R ignores it, the E column there is 1
      float4 hi, lo;
      tc::split_tf32(v[0], hi.x, lo.x);
      tc::split_tf32(v[1], hi.y, lo.y);
      tc::split_tf32(v[2], hi.z, lo.z);
      tc::split_tf32(v[3], hi.w, lo.w);
      const uint32_t off = tc::kmajor_offset(o1, 4 * p, kC) / 4;
      *reinterpret_cast<float4*>(&sm.zt[4 * i + q][0][off]) = hi;
      *reinterpret_cast<float4*>(&sm.zt[4 * i + q][1][off]) = lo;
    }
  };
  // ky pairs g, g + 2, g + 4 of unit u in fragment sets a0, a1, a2 (fills 3 u, 3 u + 1, 3 u + 2), read during unit
  // u - 1's GEMM2 (unit 0: here)
  uint32_t a0[2][kImgK / 8][4], a1[2][kImgK / 8][4], a2[2][kImgK / 8][4];
  auto first_pair = [&](uint32_t (&a)[2][kImgK / 8][4], int f) {
    load_pair(a, f);
    tc::named_barrier(2 + g, 128);   // all 128 threads have read fill f
    if (t == 0 && f + 1 < n_yfills) y_fill(f + 1);
  };
  if (n_units > 0) {
    first_pair(a0, 0);
    first_pair(a1, 1);
    first_pair(a2, 2);
  }

  for (int u = 0; u < n_units; ++u) {
    const int b = b0 + u * bstride;
    const bool more = u + 1 < n_units;
    // ---------------------------------------------------------------- GEMM1: ky pairs g, g + 2, g + 4
    float acc1[2][16];
    issue_pair(acc1[0], a0);
    issue_pair(acc1[1], a1);
    tc::wg_wait<1>();   // pair g
    tc::wg_fence_acc(acc1[0]);
    tc::named_barrier(1, 256);   // both warpgroups are done with the previous unit's Zt
    store_pair(acc1[0], g);
    issue_pair(acc1[0], a2);
    tc::wg_wait<1>();   // pair g + 2
    tc::wg_fence_acc(acc1[1]);
    store_pair(acc1[1], g + 2);
    tc::wg_wait<0>();   // pair g + 4: a0, a1, a2 are free
    tc::wg_fence_acc(acc1[0]);
    store_pair(acc1[0], g + 4);
    tc::fence_proxy_async_smem();
    tc::named_barrier(1, 256);   // Zt of all 16 rows is complete

    // ---------------------------------------------------------------- GEMM2: rows g, g + 2, ..., 14 + g
    // Iteration r issues row r's MMAs into acc[r & 1], then finishes row r - 1: wait for its MMAs (all but the newest
    // group), GELU into staging tile (r - 1) & 1, one TMA store, and the refill of the activation slot it read.
    // The MMAs read x_frag[r & 1] from registers until that wait, so the next row loads into the other set.
    float acc[2][16];
    uint32_t x_frag[2][kC / 16][4];
#pragma unroll
    for (int r = 0; r <= kFzWgRows; ++r) {
      if (r < kFzWgRows) {
        const int n = kFzWgRows * u + r, hl = g + 2 * r;
        mbar_wait(&sm.x_full[g][fz_x_slot(n)], fz_x_parity(n));
        // A[m = w][k = i] of K step ks from lines i of the slot: matrix j = lines 16 ks + 8 (j >> 1) .. + 7, pixels
        // 16 wq + 8 (j & 1) .. + 7 (one 16-byte chunk per line, distinct swizzle phases: no bank conflicts)
        const uint32_t a_x = tc::smem_addr(sm.x[g][fz_x_slot(n)]);
#pragma unroll
        for (int ks = 0; ks < kC / 16; ++ks)
          tc::ldmatrix_x4_trans(x_frag[r & 1][ks], a_x + sw128_bf16_offset(16 * ks + 8 * (lane >> 4) + (lane & 7),
                                                                             16 * wq + 8 * ((lane >> 3) & 1)));
        tc::wg_fence();
        const uint32_t b_z[3] = {tc::smem_addr(sm.zt[hl][0]), tc::smem_addr(sm.zt[hl][0]), tc::smem_addr(sm.zt[hl][1])};
#pragma unroll
        for (int pass = 0; pass < 3; ++pass)   // E_hi Zt_hi + E_lo Zt_hi + E_hi Zt_lo
#pragma unroll
          for (int ks = 0; ks < kZK / 8; ++ks)
            tc::wg_tf32_rs_n32(acc[r & 1], e_frag[pass == 1][ks],
                               tc::make_smem_desc(b_z[pass] + ks * 2 * kLboO, kLboO, 128), (pass | ks) ? 1u : 0u);
        tc::wg_fence();   // the bf16 MMAs below have another shape: order their accumulator accesses explicitly
#pragma unroll
        for (int term = 0; term < 3; ++term)
#pragma unroll
          for (int ks = 0; ks < kC / 16; ++ks)   // K = 16 channels
            tc::wg_bf16_rs_n32(acc[r & 1], x_frag[r & 1][ks],
                               tc::make_smem_desc(w0_s + term * kFzW0Bytes + ks * 2 * kLboO, kLboO, 128), 1u);
        tc::wg_commit();
        // the next unit's image fragments, one ky pair every other row (fill 3 u + 3 + r / 2); the row barrier below
        // frees the slot for the next fill, which then has two rows to land
        if (more && r == 1) load_pair(a0, 3 * u + 3);
        if (more && r == 3) load_pair(a1, 3 * u + 4);
        if (more && r == 5) load_pair(a2, 3 * u + 5);
      }
      if (r == 0) continue;
      const int rr = r - 1, h = kFzRows * chunk + g + 2 * rr;
      float* d = acc[rr & 1];
      if (r < kFzWgRows) {
        tc::wg_wait<1>();
      } else {
        tc::wg_wait<0>();
      }
      tc::wg_fence_acc(acc[rr & 1]);
      // d[4 i + 2 hh + e] = D[w = m0 + 8 hh][o = 8 i + 2 q + e] -> staging line o, element w.  The pair e = 0, 1 is one
      // bf16x2 register of the transposed 8x8 matrix (i, hh): its rows are lines 8 i .. 8 i + 7, each one 16-byte chunk
      // at pixel 16 wq + 8 hh.  Eight lines have distinct swizzle phases: no bank conflicts.
      unsigned char* stile = sm.st[g][rr & 1];
#pragma unroll
      for (int i2 = 0; i2 < 2; ++i2) {   // matrix j of the x4 store: i = 2 i2 + (j >> 1), hh = j & 1
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int i = 2 * i2 + (j >> 1), hh = j & 1;
          const float2 y = gelu_erf2(make_float2(d[4 * i + 2 * hh], d[4 * i + 2 * hh + 1]));
          const __nv_bfloat162 p = __floats2bfloat162_rn(y.x, y.y);
          v[j] = *reinterpret_cast<const uint32_t*>(&p);
        }
        tc::stmatrix_x4_trans(tc::smem_addr(stile) + sw128_bf16_offset(16 * i2 + 8 * (lane >> 4) + (lane & 7),
                                                                       16 * wq + 8 * ((lane >> 3) & 1)),
                              v);
      }
      tc::fence_proxy_async_smem();
      // the store of the previous row has read its tile, which the next row's epilogue overwrites
      if (t == 0) bulk_wait_group_read<0>();
      // all 128 threads: tile written, and row rr's MMAs -- the last readers of its activation slot -- complete
      tc::named_barrier(2 + g, 128);
      if (t == 0) {
        tma_store_3d(&out_map, stile, 0, h, b * kC);
        bulk_commit_group();
        const int nf = kFzWgRows * u + rr + kFzXSlots;
        if (nf < n_fills) x_fill(nf);
        // all 128 threads have read image fill 3 u + 3 + r / 2 (this row's loads precede the barrier above)
        if (more && (r == 1 || r == 3 || r == 5) && 3 * u + 4 + (r >> 1) < n_yfills) y_fill(3 * u + 4 + (r >> 1));
      }
    }
  }
  if (t == 0) bulk_wait_group<0>();   // the staging tiles live in this CTA's shared memory
}

// ------------------------------------------------------------------------------------------------
// Constant tables, built once per device in float64 and split into tf32 hi/lo (round to nearest).
//   etab: the C2R operand of fno_block_tc.cu with c_ky/HW folded in (c_0 = 1, c_ky = 2: Hermitian fold).
//   ftab: per chunk c, B operand of GEMM1 [n = 2 h' + ri (32)][k = 24 (kxi & 1) + 2 (kxi >> 1) + ri' (48)], h = 16 c + h',
//         kx = kxi (< 12) or kxi + 40: (ri,ri') = (0,0): cos t, (0,1): -sin t, (1,0): sin t, (1,1): cos t,
//         t = 2 pi kx h/64;  K-major hi image | lo image.
// ------------------------------------------------------------------------------------------------
void c2r_operand_table(float* host, double s0, double s1);

struct FzTables {
  float* etab = nullptr;
  float* ftab = nullptr;
  int n_sm = 0;
  bool configured = false;
};
static FzTables g_fz[64];

static cudaError_t fz_ensure(int dev, cudaStream_t stream) {
  FzTables& t = g_fz[dev];
  if (t.configured) return cudaSuccess;
  const double two_pi = 6.283185307179586476925286766559;
  static float h_e[kFzEFloats];
  static float h_f[kFzChunks * kFzFFloats];
  c2r_operand_table(h_e, 1.0 / kHW, 2.0 / kHW);
  for (int c = 0; c < kFzChunks; ++c)
    for (int n = 0; n < 2 * kFzRows; ++n) {
      const int h = kFzRows * c + (n >> 1), ri = n & 1;
      for (int k = 0; k < kImgK; ++k) {
        const int rip = k & 1, kxi = 2 * ((k % 24) >> 1) + k / 24, kx = kxi < kM1 ? kxi : kxi + (kH - kKX);
        const double ang = two_pi * ((kx * h) % 64) / 64.0;
        const double val = (ri == rip) ? cos(ang) : (ri == 0 ? -sin(ang) : sin(ang));
        const float hi = tc::round_tf32(static_cast<float>(val));
        const uint32_t off = tc::kmajor_offset(n, k, 2 * kFzRows) / 4;
        h_f[c * kFzFFloats + off] = hi;
        h_f[c * kFzFFloats + kFzFFloats / 2 + off] = tc::round_tf32(static_cast<float>(val - static_cast<double>(hi)));
      }
    }
  cudaError_t e = cudaMalloc(&t.etab, sizeof(h_e));
  if (e != cudaSuccess) return e;
  e = cudaMalloc(&t.ftab, sizeof(h_f));
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.etab, h_e, sizeof(h_e), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.ftab, h_f, sizeof(h_f), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return e;
  e = cudaStreamSynchronize(stream);   // the host arrays are static
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(block_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FzSmem));
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&t.n_sm, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  t.configured = true;
  return cudaSuccess;
}

void block_fused_release(int dev) {
  if (dev < 0 || dev >= 64) return;
  FzTables& t = g_fz[dev];
  if (t.etab) cudaFree(t.etab);
  if (t.ftab) cudaFree(t.ftab);
  t = FzTables();
}

cudaError_t launch_block_fused(const void* ym_img, const void* x, const float* w0t, const float* bias, void* out, int batch,
                               cudaStream_t stream) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  e = fz_ensure(dev, stream);
  if (e != cudaSuccess) return e;
  // TMA needs 16-byte aligned global addresses
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(ym_img) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return cudaErrorMisalignedAddress;
  // x and out as [batch * 32 planes][64 h][64 w] bf16; box = one image row of the 32 channels of a sample.  The maps are
  // kernel parameters, so a captured graph keeps the ones of its own buffers.
  CUtensorMap x_map, out_map;
  const uint64_t planes = static_cast<uint64_t>(batch) * kC;
  e = make_tma_map_3d(&x_map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, kW, kH, planes, kFzBoxW, kFzBoxH, kFzBoxC);
  if (e != cudaSuccess) return e;
  e = make_tma_map_3d(&out_map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out, kW, kH, planes, kFzBoxW, kFzBoxH, kFzBoxC);
  if (e != cudaSuccess) return e;
  // four CTAs (one per chunk of rows) per sample slot; the slots stride over the batch
  const int slots_max = g_fz[dev].n_sm / kFzChunks;
  const int slots = batch < slots_max ? batch : slots_max;
  return launch_chained(block_fused_kernel, dim3(kFzChunks * slots), dim3(kFzThreads), sizeof(FzSmem), stream, x_map,
                        out_map, static_cast<const unsigned char*>(ym_img), w0t, bias,
                        static_cast<const float*>(g_fz[dev].etab), static_cast<const float*>(g_fz[dev].ftab), batch);
}

}  // namespace fno
