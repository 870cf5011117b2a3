// K1 -- truncated forward 2-D DFT of fp32 planes: x[b][c][64][64] -> Xm[b][k][c] (288 modes).  Runs the fp32-storage
// forward and every gradient plane of the backward; bf16 planes go through dft_fwd_tc_kernel (fno_dft_fwd_tc.cu).
//
// Replaces torch.fft.rfft2 + the two corner slices of the reference
// (src/models/fno/fno2d.py:62,73-78): only kx in {0..11, 52..63} x ky in {0..11} is ever used, so
// the full 64x33 spectrum (138 MB at B=256) is never materialised.
//
// One CTA = 4 consecutive (b,c) planes = one contiguous 64 KB (fp32) run of the NCHW tensor, pulled
// into shared memory by a single bulk copy (TMA engine).  Stage 1: thread (plane, w) runs a pruned
// real 64-point DFT down column w in registers (bins kx' = 0..12; Hermitian symmetry supplies the
// negative rows).  Stage 2: each of the 13 complex rows per plane is transformed along w by 4
// threads, thread j producing the bins = j (mod 4) of {-11..11} (DIF split, no exchange needed);
// j is warp-uniform so the four codelets do not diverge.  X[64-kx', ky] = conj(F[kx'][-ky]).
#include "fft_codelets.cuh"
#include "fno_common.cuh"

namespace fno {

constexpr int kDftPlanes = 2;     // planes per CTA (small CTAs: 4-5 resident per SM hide each other's TMA wait)
constexpr int kDftMinBlocks = 4;  // resident CTAs per SM the kernel is compiled for
constexpr int kDftThreads = 128;  // 64 columns x 2 planes
constexpr int kDftRows = kDftPlanes * 13;
constexpr int kDftRowPitch = 65;  // float2 elements; +1 keeps stage-2 row gathers conflict-free

struct DftSmem {
  alignas(128) float xs[kDftPlanes * kHW];
  alignas(16) float2 as[kDftRows * kDftRowPitch];
  alignas(8) uint64_t bar;
};

// bins (in codelet output order) produced by cfft64_r<J>: the members of {0..11, 53..63} that are = J mod 4
template <int J>
__host__ __device__ constexpr int fwd_bin_count() {
  return J == 0 ? 5 : 6;
}
template <int J>
__host__ __device__ constexpr int fwd_bin(int e) {
  return e < 3 ? 4 * e + J : (J == 0 ? 4 * e + 44 : 4 * e + J + 40);
}

template <int J>
__device__ __forceinline__ void row_transform_and_emit(const float2* __restrict__ row, float2* __restrict__ xm_b,
                                                       size_t mode_stride,
                                                       int kxp, int c, float s0, float s1) {
  float xre[64], xim[64], ore[6], oim[6];
#pragma unroll
  for (int n = 0; n < 64; ++n) {
    const float2 v = row[n];
    xre[n] = v.x;
    xim[n] = v.y;
  }
  if constexpr (J == 0) fno_codelets::cfft64_r0<float>(xre, xim, ore, oim);
  if constexpr (J == 1) fno_codelets::cfft64_r1<float>(xre, xim, ore, oim);
  if constexpr (J == 2) fno_codelets::cfft64_r2<float>(xre, xim, ore, oim);
  if constexpr (J == 3) fno_codelets::cfft64_r3<float>(xre, xim, ore, oim);
#pragma unroll
  for (int e = 0; e < fwd_bin_count<J>(); ++e) {
    const int q = fwd_bin<J>(e);
    if (q <= 11) {  // X[kx', q] = F[kx'][q], rows 0..11 (weights1 block)
      if (kxp <= 11) {
        const float s = (q == 0) ? s0 : s1;
        xm_b[(kxp * kM2 + q) * mode_stride + c] = make_float2(ore[e] * s, oim[e] * s);
      }
    }
    const int qq = (64 - q) & 63;
    if (qq <= 11) {  // X[64-kx', qq] = conj(F[kx'][-qq]), rows 52..63 (weights2 block)
      if (kxp >= 1) {
        const float s = (qq == 0) ? s0 : s1;
        xm_b[((kKX - kxp) * kM2 + qq) * mode_stride + c] = make_float2(ore[e] * s, -oim[e] * s);
      }
    }
  }
}

__global__ void __launch_bounds__(kDftThreads, kDftMinBlocks)
    dft_fwd_kernel(const float* __restrict__ x, float2* __restrict__ xm, float s0, float s1) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  DftSmem& sm = *reinterpret_cast<DftSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int plane0 = blockIdx.x * kDftPlanes;  // global plane index = b*32 + c
  const int b = plane0 / kC;
  const int c0 = plane0 % kC;

  if (tid == 0) {
    mbar_init(&sm.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  if (tid == 0) {
    constexpr uint32_t bytes = kDftPlanes * kHW * sizeof(float);
    mbar_expect_tx(&sm.bar, bytes);
    bulk_g2s(sm.xs, x + static_cast<size_t>(plane0) * kHW, bytes, &sm.bar);
  }
  mbar_wait(&sm.bar, 0);

  // ---- stage 1: real DFT along h, one thread per (plane, column w) --------------------------
  {
    const int p = tid >> 6, w = tid & 63;
    float v[64], ore[13], oim[13];
    const float* col = sm.xs + p * kHW + w;
#pragma unroll
    for (int h = 0; h < 64; ++h) v[h] = col[h * kW];
    fno_codelets::rfft64_lo13<float>(v, ore, oim);
    float2* dst = sm.as + (p * 13) * kDftRowPitch + w;
#pragma unroll
    for (int k = 0; k < 13; ++k) dst[k * kDftRowPitch] = make_float2(ore[k], oim[k]);
  }
  __syncthreads();

  // ---- stage 2: complex DFT along w, 4 threads (j = warp & 3) per row ----------------------
  {
    const int warp = tid >> 5, lane = tid & 31;
    const int j = warp & 3;
    const int rho = (warp >> 2) * 26 + lane;  // row index p*13 + kx'
    if (lane < 26) {
      const int p = rho / 13, kxp = rho % 13;
      const float2* row = sm.as + rho * kDftRowPitch;
      // modes are stored mode-major, xm[k][b][c]: the mix reads one mode of a whole sample tile as one contiguous block
      const size_t mode_stride = static_cast<size_t>(gridDim.x) * kDftPlanes;  // = batch * kC float2 per mode
      float2* xm_b = xm + static_cast<size_t>(b) * kC;
      const int c = c0 + p;
      switch (j) {
        case 0: row_transform_and_emit<0>(row, xm_b, mode_stride, kxp, c, s0, s1); break;
        case 1: row_transform_and_emit<1>(row, xm_b, mode_stride, kxp, c, s0, s1); break;
        case 2: row_transform_and_emit<2>(row, xm_b, mode_stride, kxp, c, s0, s1); break;
        default: row_transform_and_emit<3>(row, xm_b, mode_stride, kxp, c, s0, s1); break;
      }
    }
  }
}

cudaError_t launch_dft_fwd(const void* x, void* xm, int batch, float s0, float s1, cudaStream_t stream) {
  constexpr size_t smem = sizeof(DftSmem);
  static PerDeviceLaunch pd;
  cudaError_t e0 = per_device_setup(dft_fwd_kernel, smem, pd);
  if (e0 != cudaSuccess) return e0;
  const int n_ctas = batch * kC / kDftPlanes;
  return launch_chained(dft_fwd_kernel, dim3(n_ctas), dim3(kDftThreads), smem, stream, static_cast<const float*>(x),
                        static_cast<float2*>(xm), s0, s1);
}

}  // namespace fno
