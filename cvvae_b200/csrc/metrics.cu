// Reconstruction quality on the device: per-frame squared error and SSIM of two uint8 videos [T,H,W,3], the two ends of
// the inference script (its resized input, cvvae_inference_video.py:28, and its uint8 output, :47-50).
//
// SSIM is Wang et al. 2004 with the 11-tap Gaussian window (sigma 1.5, normalised), population covariance, data range
// 255, per colour channel, over the positions whose window lies inside the frame (5-pixel border cropped, no padding).
//
// A frame is an image of H rows x 3W bytes, and a colour channel's horizontal neighbours are 3 bytes apart, so the
// window is an 11 x 11 filter with a horizontal dilation of 3 on that byte image and the channels need no special care.
// One CTA scores a patch of kMetRows x kMetThreads output bytes.  It walks down the patch 11 input rows at a time:
// the rows (with their 15-byte halo either side) are staged in shared memory by 16-byte loads, every thread runs the
// horizontal pass of its column over the five moment maps (a, b, a^2, b^2, ab) and keeps the last 11 rows of them in
// registers, and each new row completes the vertical pass of one output row.  No map ever leaves the SM; global
// traffic is one read of each frame plus the halo overlap.
//
// The moments are computed on pixel values shifted by -128 (variances and the covariance are shift-invariant; the means
// get the shift back).  fp32 is not enough for them: E[a^2] reaches 2^14, where fp32 resolves 2^-10, and C2 = 58.5 turns
// the dozen roundings of a flat 255-against-254 window into an SSIM error of 8e-5.  So the horizontal pass is exact
// integer arithmetic (weights as multiples of 2^-32 that sum to exactly 1, 64-bit sums) and the vertical pass is fp64
// FMAs, which this GPU issues at half the fp32 rate; the central moments are rounded to fp32 once and the formula is
// evaluated in fp32, symmetrically and with explicit roundings, so identical frames give exactly 1.0 at every position.
// Per-position SSIM is rounded to 2^-32 and summed, like the squared error, in 64-bit integers (warp shuffles, one
// atomic pair per CTA): the result is independent of the summation order, hence of the grid, and bit-reproducible.
#include <math.h>

#include "common.cuh"

namespace cvvae {

constexpr int kMetThreads = 128;                                  // output byte-columns per CTA, one thread each
constexpr int kMetRows = 44;                                      // output rows per CTA
constexpr int kMetTaps = 11;
constexpr int kMetHaloBytes = 3 * (kMetTaps / 2);                 // 15 bytes = 5 pixels either side
constexpr int kMetPatchBytes = kMetThreads + 2 * kMetHaloBytes;   // bytes of one staged row that are used
constexpr int kMetVecs = (kMetPatchBytes + 15 + 15) / 16;         // 16-byte vectors covering them at any misalignment
constexpr int kMetPitch = kMetVecs * 16;

// The window's weights g[k] = exp(-(k-5)^2 / (2 * 1.5^2)) / sum as multiples of 2^-32 that add up to exactly 1: q = g * 2^32.
struct MetWeights {
  double g[kMetTaps];
  int q[kMetTaps];
};

// The 16 bytes at `q` (16-byte aligned).  A vector that reaches outside the tensor [lo, hi) - only the first and the last
// one of the whole video can - is read byte by byte, the bytes outside as 0 (they are never used).
__device__ __forceinline__ uint4 load_vec16(uintptr_t q, uintptr_t lo, uintptr_t hi) {
  if (q >= lo && q + 16 <= hi) return __ldg(reinterpret_cast<const uint4*>(q));
  uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int i = 0; i < 16; ++i)
    if (q + i >= lo && q + i < hi) w[i >> 2] |= static_cast<uint32_t>(*reinterpret_cast<const uint8_t*>(q + i)) << (8 * (i & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__global__ void __launch_bounds__(kMetThreads)
    frame_metrics_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int H, int WB, int tiles_x, int chunks_y,
                         long long total_bytes, MetWeights wt, unsigned long long* __restrict__ acc) {
  // rows of the open group, as int8 = pixel - 128 (stored as pixel ^ 0x80), each at its global 16-byte alignment:
  // byte i of the patch row sits at s_px[frame][row][s_mis[frame][row] + i]
  __shared__ __align__(16) uint8_t s_px[2][kMetTaps][kMetPitch];
  __shared__ int s_mis[2][kMetTaps];
  __shared__ unsigned long long s_red[kMetThreads / 32][2];

  const int tile = blockIdx.x % tiles_x;
  const int chunk = (blockIdx.x / tiles_x) % chunks_y;
  const int t = blockIdx.x / (tiles_x * chunks_y);
  // Output column c (0 <= c < WB - 30) is centred on byte c + 15 of the row and reads bytes [c, c + 30]; likewise rows.
  const int c0 = tile * kMetThreads, r0 = chunk * kMetRows;
  const int ncols = min(kMetThreads, WB - 2 * kMetHaloBytes - c0);
  const int nrows_in = min(kMetRows, H - (kMetTaps - 1) - r0) + kMetTaps - 1;
  const int nbytes = ncols + 2 * kMetHaloBytes;
  // The squared error covers the whole frame: every byte is counted by the one CTA whose outputs are centred on it,
  // and the CTAs along the frame's edges take the border with them.
  const int own_c_lo = tile == 0 ? 0 : kMetHaloBytes;
  const int own_c_hi = kMetHaloBytes + ncols + (tile == tiles_x - 1 ? kMetHaloBytes : 0);
  const int own_r_lo = chunk == 0 ? 0 : kMetTaps / 2;
  const int own_r_hi = nrows_in - (chunk == chunks_y - 1 ? 0 : kMetTaps / 2);

  const uintptr_t base_a = reinterpret_cast<uintptr_t>(a), base_b = reinterpret_cast<uintptr_t>(b);
  const long long patch_off = (static_cast<long long>(t) * H + r0) * WB + c0;

  double ring[5][kMetTaps];   // horizontal-pass results of the last 11 rows, times 2^32: sums of a, b, a^2, b^2, ab
  unsigned long long sse = 0;
  long long ssim_fix = 0;

  for (int g0 = 0; g0 < nrows_in; g0 += kMetTaps) {
    const int nr = min(kMetTaps, nrows_in - g0);
    __syncthreads();   // the previous group has been consumed
    for (int item = threadIdx.x; item < 2 * nr * kMetVecs; item += kMetThreads) {
      const int v = item % kMetVecs, fr = item / kMetVecs;
      const int f = fr >= nr ? 1 : 0, row = fr - f * nr;
      const uintptr_t base = f ? base_b : base_a;
      const uintptr_t p = base + static_cast<uintptr_t>(patch_off + static_cast<long long>(g0 + row) * WB);
      const int mis = static_cast<int>(p & 15);
      if (v == 0) s_mis[f][row] = mis;
      if (v * 16 < mis + nbytes) {
        uint4 x = load_vec16(p - mis + v * 16, base, base + static_cast<uintptr_t>(total_bytes));
        x.x ^= 0x80808080u;
        x.y ^= 0x80808080u;
        x.z ^= 0x80808080u;
        x.w ^= 0x80808080u;
        *reinterpret_cast<uint4*>(&s_px[f][row][v * 16]) = x;
      }
    }
    __syncthreads();

    for (int row = 0; row < nr; ++row) {
      if (g0 + row < own_r_lo || g0 + row >= own_r_hi) continue;
      const int8_t* pa = reinterpret_cast<const int8_t*>(s_px[0][row]) + s_mis[0][row];
      const int8_t* pb = reinterpret_cast<const int8_t*>(s_px[1][row]) + s_mis[1][row];
      for (int c = own_c_lo + threadIdx.x; c < own_c_hi; c += kMetThreads) {
        const int d = static_cast<int>(pa[c]) - static_cast<int>(pb[c]);
        sse += static_cast<unsigned>(d * d);
      }
    }

    if (static_cast<int>(threadIdx.x) < ncols) {
#pragma unroll
      for (int j = 0; j < kMetTaps; ++j) {
        if (j < nr) {
          const int8_t* pa = reinterpret_cast<const int8_t*>(s_px[0][j]) + s_mis[0][j] + threadIdx.x;
          const int8_t* pb = reinterpret_cast<const int8_t*>(s_px[1][j]) + s_mis[1][j] + threadIdx.x;
          long long h[5] = {0, 0, 0, 0, 0};   // exact: |sum| <= 2^32 * 128^2
#pragma unroll
          for (int k = 0; k < kMetTaps; ++k) {
            const int x = pa[3 * k], y = pb[3 * k];
            h[0] += static_cast<long long>(wt.q[k]) * x;
            h[1] += static_cast<long long>(wt.q[k]) * y;
            h[2] += static_cast<long long>(wt.q[k]) * (x * x);
            h[3] += static_cast<long long>(wt.q[k]) * (y * y);
            h[4] += static_cast<long long>(wt.q[k]) * (x * y);
          }
#pragma unroll
          for (int q = 0; q < 5; ++q) ring[q][j] = static_cast<double>(h[q]);   // exact (below 2^53)
          if (g0 + j >= kMetTaps - 1) {   // rows g0+j-10 .. g0+j are in the ring: one output row is complete
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < kMetTaps; ++k) {
              const int slot = (j + 1 + k) % kMetTaps;   // ring slot of row g0+j-10+k
#pragma unroll
              for (int q = 0; q < 5; ++q) m[q] = fma(wt.g[k], ring[q][slot], m[q]);
            }
#pragma unroll
            for (int q = 0; q < 5; ++q) m[q] *= 1.0 / 4294967296.0;
            // The three central moments are the same expression of their inputs, and so is each side of the fraction:
            // identical frames give va == vb == vab, num == den and a quotient of exactly 1.
            const float va = static_cast<float>(fma(-m[0], m[0], m[2]));
            const float vb = static_cast<float>(fma(-m[1], m[1], m[3]));
            const float vab = static_cast<float>(fma(-m[0], m[1], m[4]));
            const float mua = static_cast<float>(m[0] + 128.0), mub = static_cast<float>(m[1] + 128.0);
            const float c1 = 6.5025f, c2 = 58.5225f;
            const float pab = __fmul_rn(mua, mub);
            const float lum_n = __fadd_rn(__fadd_rn(pab, pab), c1);
            const float lum_d = __fadd_rn(__fadd_rn(__fmul_rn(mua, mua), __fmul_rn(mub, mub)), c1);
            const float cs_n = __fadd_rn(__fadd_rn(vab, vab), c2);
            const float cs_d = __fadd_rn(__fadd_rn(va, vb), c2);
            const float ssim = __fdiv_rn(__fmul_rn(lum_n, cs_n), __fmul_rn(lum_d, cs_d));
            ssim_fix += __float2ll_rn(ssim * 4294967296.f);
          }
        }
      }
    }
  }

  unsigned long long fix = static_cast<unsigned long long>(ssim_fix);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sse += __shfl_down_sync(0xffffffffu, sse, o);
    fix += __shfl_down_sync(0xffffffffu, fix, o);
  }
  if ((threadIdx.x & 31) == 0) {
    s_red[threadIdx.x >> 5][0] = sse;
    s_red[threadIdx.x >> 5][1] = fix;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned long long s = 0;
#pragma unroll
    for (int w = 0; w < kMetThreads / 32; ++w) s += s_red[w][threadIdx.x];
    atomicAdd(acc + 2 * static_cast<size_t>(t) + threadIdx.x, s);
  }
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_frame_metrics(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, int64_t* acc,
                                   void* stream_) {
  CVVAE_CHECK_ARG(a_thwc && b_thwc && acc, "cvvae_frame_metrics: null pointer");
  CVVAE_CHECK_ARG(T >= 0 && H >= kMetTaps && W >= kMetTaps,
                  "cvvae_frame_metrics: needs T >= 0 and frames of at least 11 x 11 px, got T=%d H=%d W=%d", (int)T, (int)H, (int)W);
  // sum over 3*H*W positions of ssim * 2^32 must stay inside int64
  CVVAE_CHECK_ARG(3ll * H * W < (1ll << 31), "cvvae_frame_metrics: %d x %d frames exceed the 64-bit accumulator's range (3*H*W < 2^31)",
                  (int)H, (int)W);
  if (T == 0) return CVVAE_OK;
  const int WB = 3 * W;
  const int tiles_x = (WB - 2 * kMetHaloBytes + kMetThreads - 1) / kMetThreads;
  const int chunks_y = (H - (kMetTaps - 1) + kMetRows - 1) / kMetRows;
  const long long grid = 1ll * tiles_x * chunks_y * T;
  CVVAE_CHECK_ARG(grid < (1ll << 31), "cvvae_frame_metrics: too many frames for one launch (T=%d at %d x %d)", (int)T, (int)H, (int)W);

  MetWeights wt;   // the centre tap absorbs the rounding of the others
  double g[kMetTaps], sum = 0.0;
  for (int k = 0; k < kMetTaps; ++k) sum += g[k] = exp(-(k - 5) * (k - 5) / 4.5);
  long long rest = 1ll << 32;
  for (int k = 0; k < kMetTaps; ++k) rest -= wt.q[k] = static_cast<int>(llrint(g[k] / sum * 4294967296.0));
  wt.q[kMetTaps / 2] += static_cast<int>(rest);
  for (int k = 0; k < kMetTaps; ++k) wt.g[k] = wt.q[k] / 4294967296.0;

  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_CUDA(cudaMemsetAsync(acc, 0, sizeof(int64_t) * 2 * T, stream));
  frame_metrics_kernel<<<static_cast<unsigned>(grid), kMetThreads, 0, stream>>>(
      a_thwc, b_thwc, H, WB, tiles_x, chunks_y, 1ll * T * H * WB, wt, reinterpret_cast<unsigned long long*>(acc));
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
