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
//
// MS-SSIM (cvvae_frame_ms_ssim) runs the same kernel at five scales.  Level j+1 is the 2x2 average pool of level j (an
// odd extent is zero-padded in front, as pytorch_msssim does); a level-j pixel is an integer sum of at most 4^j bytes
// divided by 4^j, so the levels are stored as those sums in uint16 (at most 255 * 4^4 = 65280) and are exact.  The
// scoring kernel reads them as they are: shifted by -128 * 4^j they stay within 2^15, so the horizontal pass's
// sum q_k x^2 stays below 2^62 and is still exact in int64; the formula is evaluated in level-j sum units, with C1 and C2
// scaled by 16^j (a power of two, so no fp32 rounding changes).  In this mode a CTA
// leaves, per colour channel, the sums of cs = (2 s_ab + C2) / (s_a^2 + s_b^2 + C2) and of the full SSIM, in units of
// 2^-32; the channel of an output column is its element column mod 3.
//
// The SSIM map (cvvae_frame_ssim_map) is the byte instantiation with MAP set: every output element also stores its fp32
// ssim, the value it rounds and sums, at map[t][r][c] with c its element column, so the map holds exactly the terms of the
// frame's SSIM sum.  Consecutive threads own consecutive columns, so the stores of a row are coalesced.
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace cvvae {

constexpr int kMetThreads = 128;                            // output element-columns per CTA, one thread each
constexpr int kMetRows = 44;                                // output rows per CTA
constexpr int kMetTaps = 11;
constexpr int kMetHalo = 3 * (kMetTaps / 2);                // 15 elements = 5 pixels either side
constexpr int kMetPatch = kMetThreads + 2 * kMetHalo;       // elements of one staged row that are used
constexpr int kMsLevels = 5;                                // MS-SSIM scales
constexpr int kMsMinSize = 160;                             // MS-SSIM needs frames larger than this: level 4 holds the window
// 16-byte vectors covering one staged row of E at any misalignment
template <typename E>
constexpr int met_vecs() {
  return (kMetPatch * static_cast<int>(sizeof(E)) + 15 + 15) / 16;
}

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

// E: uint8_t (frames) or uint16_t (MS-SSIM levels >= 1, sums of 4^j pixels); a row of a frame is WE = 3W elements.
// MS false (cvvae_frame_metrics): acc[t] += {squared error, SSIM}.  MS true (one level of cvvae_frame_ms_ssim):
// acc[t * 30 + 2 c] += {cs, SSIM} of channel c, with the elements shifted by `shift` = 128 * 4^j and C1, C2 = c1s, c2s.
// MAP (bytes, MS false; cvvae_frame_ssim_map): also map[(t (H - 10) + r) (WE - 30) + c] = ssim of output element (r, c).
template <typename E, bool MS, bool MAP = false>
__global__ void __launch_bounds__(kMetThreads)
    frame_metrics_kernel(const E* __restrict__ a, const E* __restrict__ b, int H, int WE, int tiles_x, int chunks_y,
                         long long total_bytes, MetWeights wt, unsigned long long* __restrict__ acc, int shift, float c1s,
                         float c2s, float* __restrict__ map) {
  static_assert(!MAP || (sizeof(E) == 1 && !MS), "the SSIM map is the byte, non-MS instantiation");
  using S = typename std::conditional<sizeof(E) == 1, int8_t, int16_t>::type;   // staged: element - shift
  constexpr int kVecs = met_vecs<E>(), kPitch = kVecs * 16;
  // rows of the open group, as element - shift (for bytes: stored as pixel ^ 0x80), each at its global 16-byte alignment:
  // element i of the patch row sits at byte s_mis[frame][row] + i * sizeof(E) of s_px[frame][row]
  __shared__ __align__(16) uint8_t s_px[2][kMetTaps][kPitch];
  __shared__ int s_mis[2][kMetTaps];
  __shared__ unsigned long long s_red[kMetThreads / 32][MS ? 6 : 2];

  const int tile = blockIdx.x % tiles_x;
  const int chunk = (blockIdx.x / tiles_x) % chunks_y;
  const int t = blockIdx.x / (tiles_x * chunks_y);
  // Output column c (0 <= c < WE - 30) is centred on element c + 15 of the row and reads elements [c, c + 30]; likewise rows.
  const int c0 = tile * kMetThreads, r0 = chunk * kMetRows;
  const int ncols = min(kMetThreads, WE - 2 * kMetHalo - c0);
  const int nrows_in = min(kMetRows, H - (kMetTaps - 1) - r0) + kMetTaps - 1;
  const int nbytes = (ncols + 2 * kMetHalo) * static_cast<int>(sizeof(E));
  // The squared error covers the whole frame: every byte is counted by the one CTA whose outputs are centred on it,
  // and the CTAs along the frame's edges take the border with them.
  const int own_c_lo = tile == 0 ? 0 : kMetHalo;
  const int own_c_hi = kMetHalo + ncols + (tile == tiles_x - 1 ? kMetHalo : 0);
  const int own_r_lo = chunk == 0 ? 0 : kMetTaps / 2;
  const int own_r_hi = nrows_in - (chunk == chunks_y - 1 ? 0 : kMetTaps / 2);

  const uintptr_t base_a = reinterpret_cast<uintptr_t>(a), base_b = reinterpret_cast<uintptr_t>(b);
  const long long patch_off = (static_cast<long long>(t) * H + r0) * WE + c0;

  double ring[5][kMetTaps];   // horizontal-pass results of the last 11 rows, times 2^32: sums of a, b, a^2, b^2, ab
  unsigned long long sse = 0;
  long long ssim_fix = 0, cs_fix = 0;

  for (int g0 = 0; g0 < nrows_in; g0 += kMetTaps) {
    const int nr = min(kMetTaps, nrows_in - g0);
    __syncthreads();   // the previous group has been consumed
    for (int item = threadIdx.x; item < 2 * nr * kVecs; item += kMetThreads) {
      const int v = item % kVecs, fr = item / kVecs;
      const int f = fr >= nr ? 1 : 0, row = fr - f * nr;
      const uintptr_t base = f ? base_b : base_a;
      const uintptr_t p = base + static_cast<uintptr_t>(patch_off + static_cast<long long>(g0 + row) * WE) * sizeof(E);
      const int mis = static_cast<int>(p & 15);
      if (v == 0) s_mis[f][row] = mis;
      if (v * 16 < mis + nbytes) {
        uint4 x = load_vec16(p - mis + v * 16, base, base + static_cast<uintptr_t>(total_bytes));
        if constexpr (sizeof(E) == 1) {
          x.x ^= 0x80808080u;
          x.y ^= 0x80808080u;
          x.z ^= 0x80808080u;
          x.w ^= 0x80808080u;
        } else {   // rows start on an element, so the halfwords of the vector are elements: subtract the shift from each
          const unsigned s2 = static_cast<unsigned>(shift) * 0x10001u;
          x.x = __vsub2(x.x, s2);
          x.y = __vsub2(x.y, s2);
          x.z = __vsub2(x.z, s2);
          x.w = __vsub2(x.w, s2);
        }
        *reinterpret_cast<uint4*>(&s_px[f][row][v * 16]) = x;
      }
    }
    __syncthreads();

    if constexpr (!MS) {
      for (int row = 0; row < nr; ++row) {
        if (g0 + row < own_r_lo || g0 + row >= own_r_hi) continue;
        const int8_t* pa = reinterpret_cast<const int8_t*>(s_px[0][row]) + s_mis[0][row];
        const int8_t* pb = reinterpret_cast<const int8_t*>(s_px[1][row]) + s_mis[1][row];
        for (int c = own_c_lo + threadIdx.x; c < own_c_hi; c += kMetThreads) {
          const int d = static_cast<int>(pa[c]) - static_cast<int>(pb[c]);
          sse += static_cast<unsigned>(d * d);
        }
      }
    }

    if (static_cast<int>(threadIdx.x) < ncols) {
#pragma unroll
      for (int j = 0; j < kMetTaps; ++j) {
        if (j < nr) {
          const S* pa = reinterpret_cast<const S*>(s_px[0][j] + s_mis[0][j]) + threadIdx.x;
          const S* pb = reinterpret_cast<const S*>(s_px[1][j] + s_mis[1][j]) + threadIdx.x;
          long long h[5] = {0, 0, 0, 0, 0};   // exact: |sum| <= 2^32 * 2^30 (bytes: 2^32 * 128^2)
#pragma unroll
          for (int k = 0; k < kMetTaps; ++k) {
            const int x = pa[3 * k], y = pb[3 * k];
            h[0] += static_cast<long long>(wt.q[k]) * x;
            h[1] += static_cast<long long>(wt.q[k]) * y;
            h[2] += static_cast<long long>(wt.q[k]) * (x * x);
            h[3] += static_cast<long long>(wt.q[k]) * (y * y);
            h[4] += static_cast<long long>(wt.q[k]) * (x * y);
          }
          // exact for bytes (below 2^53); at the pooled levels the squares round to 53 bits, the same way for a and b
#pragma unroll
          for (int q = 0; q < 5; ++q) ring[q][j] = static_cast<double>(h[q]);
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
            const double sh = MS ? static_cast<double>(shift) : 128.0;
            const float mua = static_cast<float>(m[0] + sh), mub = static_cast<float>(m[1] + sh);
            const float c1 = MS ? c1s : 6.5025f, c2 = MS ? c2s : 58.5225f;
            const float pab = __fmul_rn(mua, mub);
            const float lum_n = __fadd_rn(__fadd_rn(pab, pab), c1);
            const float lum_d = __fadd_rn(__fadd_rn(__fmul_rn(mua, mua), __fmul_rn(mub, mub)), c1);
            const float cs_n = __fadd_rn(__fadd_rn(vab, vab), c2);
            const float cs_d = __fadd_rn(__fadd_rn(va, vb), c2);
            const float ssim = __fdiv_rn(__fmul_rn(lum_n, cs_n), __fmul_rn(lum_d, cs_d));
            ssim_fix += __float2ll_rn(ssim * 4294967296.f);
            if constexpr (MAP)
              map[(static_cast<long long>(t) * (H - (kMetTaps - 1)) + r0 + g0 + j - (kMetTaps - 1)) * (WE - 2 * kMetHalo) + c0 +
                  threadIdx.x] = ssim;
            if constexpr (MS) cs_fix += __float2ll_rn(__fdiv_rn(cs_n, cs_d) * 4294967296.f);
          }
        }
      }
    }
  }

  unsigned long long fix = static_cast<unsigned long long>(ssim_fix);
  if constexpr (MS) {
    // per channel: this thread's sums go to slots 2c (cs) and 2c + 1 (SSIM), the other four get zeros
    const int ch = (c0 + static_cast<int>(threadIdx.x)) % 3;
    unsigned long long v[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) v[q] = (q >> 1) != ch ? 0ull : (q & 1) ? fix : static_cast<unsigned long long>(cs_fix);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int q = 0; q < 6; ++q) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
      for (int q = 0; q < 6; ++q) s_red[threadIdx.x >> 5][q] = v[q];
    __syncthreads();
    if (threadIdx.x < 6) {
      unsigned long long s = 0;
#pragma unroll
      for (int w = 0; w < kMetThreads / 32; ++w) s += s_red[w][threadIdx.x];
      atomicAdd(acc + kMsLevels * 6 * static_cast<size_t>(t) + threadIdx.x, s);
    }
  } else {
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
}

// One MS-SSIM pooling step of both videos (blockIdx.z: a, b): dst [T, Hd, Wd, 3] = the sums of the 2 x 2 cells of
// src [T, Hs, Ws, 3].  Along an axis of even extent output i covers inputs 2i and 2i + 1; of odd extent, 2i - 1 and 2i
// with input -1 = 0 (zero padding in front, counted in the divisor 4).
template <typename E>
__global__ void __launch_bounds__(256)
    ms_pool_kernel(const E* __restrict__ sa, const E* __restrict__ sb, uint16_t* __restrict__ da, uint16_t* __restrict__ db,
                   int T, int Hs, int Ws, int Hd, int Wd) {
  const E* src = blockIdx.z ? sb : sa;
  uint16_t* dst = blockIdx.z ? db : da;
  const int n = Hd * Wd * 3;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = i % 3, px = i / 3;
  const int y0 = 2 * (px / Wd) - (Hs & 1), x0 = 2 * (px % Wd) - (Ws & 1);
  for (int t = blockIdx.y; t < T; t += gridDim.y) {
    const E* s = src + static_cast<long long>(t) * Hs * Ws * 3;
    unsigned v = 0;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx)
        if (y0 + dy >= 0 && x0 + dx >= 0) v += s[((y0 + dy) * Ws + x0 + dx) * 3 + c];
    dst[static_cast<long long>(t) * n + i] = static_cast<uint16_t>(v);
  }
}

MetWeights met_weights() {   // the centre tap absorbs the rounding of the others
  MetWeights wt;
  double g[kMetTaps], sum = 0.0;
  for (int k = 0; k < kMetTaps; ++k) sum += g[k] = exp(-(k - 5) * (k - 5) / 4.5);
  long long rest = 1ll << 32;
  for (int k = 0; k < kMetTaps; ++k) rest -= wt.q[k] = static_cast<int>(llrint(g[k] / sum * 4294967296.0));
  wt.q[kMetTaps / 2] += static_cast<int>(rest);
  for (int k = 0; k < kMetTaps; ++k) wt.g[k] = wt.q[k] / 4294967296.0;
  return wt;
}

// The scoring grid of T frames of H x W px: tiles_x * chunks_y CTAs per frame.
long long met_grid(int T, int H, int W, int* tiles_x, int* chunks_y) {
  *tiles_x = (3 * W - 2 * kMetHalo + kMetThreads - 1) / kMetThreads;
  *chunks_y = (H - (kMetTaps - 1) + kMetRows - 1) / kMetRows;
  return 1ll * *tiles_x * *chunks_y * T;
}

// Extent of MS-SSIM level j along an axis of n pixels, and the bytes of one video's level-j sums (rounded up to 256
// bytes, so that every level of the workspace starts aligned).
int ms_extent(int n, int j) {
  for (; j > 0; --j) n = (n + 1) / 2;
  return n;
}
long long ms_level_bytes(int T, int H, int W, int j) {
  return (2ll * T * ms_extent(H, j) * ms_extent(W, j) * 3 + 255) / 256 * 256;
}

// The checks and launch shared by cvvae_frame_metrics (map NULL) and cvvae_frame_ssim_map (MAP, map required).
template <bool MAP>
int frame_metrics_launch(const char* who, const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W,
                         int64_t* acc, float* map, void* stream_) {
  CVVAE_CHECK_ARG(a_thwc && b_thwc && acc && (!MAP || map), "%s: null pointer", who);
  CVVAE_CHECK_ARG(T >= 0 && H >= kMetTaps && W >= kMetTaps,
                  "%s: needs T >= 0 and frames of at least 11 x 11 px, got T=%d H=%d W=%d", who, (int)T, (int)H, (int)W);
  // sum over 3*H*W positions of ssim * 2^32 must stay inside int64
  CVVAE_CHECK_ARG(3ll * H * W < (1ll << 31), "%s: %d x %d frames exceed the 64-bit accumulator's range (3*H*W < 2^31)", who,
                  (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(map) % sizeof(float) == 0, "%s: `map` must be 4-byte aligned", who);
  if (T == 0) return CVVAE_OK;
  int tiles_x, chunks_y;
  const long long grid = met_grid(T, H, W, &tiles_x, &chunks_y);
  CVVAE_CHECK_ARG(grid < (1ll << 31), "%s: too many frames for one launch (T=%d at %d x %d)", who, (int)T, (int)H, (int)W);
  const MetWeights wt = met_weights();

  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_CUDA(cudaMemsetAsync(acc, 0, sizeof(int64_t) * 2 * T, stream));
  frame_metrics_kernel<uint8_t, false, MAP><<<static_cast<unsigned>(grid), kMetThreads, 0, stream>>>(
      a_thwc, b_thwc, H, 3 * W, tiles_x, chunks_y, 3ll * T * H * W, wt, reinterpret_cast<unsigned long long*>(acc), 128, 0.f, 0.f,
      map);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_frame_metrics(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, int64_t* acc,
                                   void* stream) {
  return frame_metrics_launch<false>("cvvae_frame_metrics", a_thwc, b_thwc, T, H, W, acc, nullptr, stream);
}

extern "C" int cvvae_frame_ssim_map(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, int64_t* acc,
                                    float* map, void* stream) {
  return frame_metrics_launch<true>("cvvae_frame_ssim_map", a_thwc, b_thwc, T, H, W, acc, map, stream);
}

extern "C" int64_t cvvae_ms_ssim_workspace_bytes(int32_t T, int32_t H, int32_t W) {
  CVVAE_CHECK_ARG(T >= 0 && H > 0 && W > 0, "cvvae_ms_ssim_workspace_bytes: needs T >= 0 and H, W >= 1, got T=%d H=%d W=%d",
                  (int)T, (int)H, (int)W);
  long long n = 0;
  for (int j = 1; j < kMsLevels; ++j) n += 2 * ms_level_bytes(T, H, W, j);
  return n;
}

extern "C" int cvvae_frame_ms_ssim(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, void* workspace,
                                   int64_t* acc, void* stream_) {
  CVVAE_CHECK_ARG(a_thwc && b_thwc && workspace && acc, "cvvae_frame_ms_ssim: null pointer");
  CVVAE_CHECK_ARG(T >= 0 && H > kMsMinSize && W > kMsMinSize,
                  "cvvae_frame_ms_ssim: needs T >= 0 and frames of at least 161 x 161 px (level 4 must hold the 11 x 11 window), "
                  "got T=%d H=%d W=%d", (int)T, (int)H, (int)W);
  CVVAE_CHECK_ARG(3ll * H * W < (1ll << 31), "cvvae_frame_ms_ssim: %d x %d frames exceed the 64-bit accumulator's range (3*H*W < 2^31)",
                  (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "cvvae_frame_ms_ssim: the workspace must be 16-byte aligned");
  if (T == 0) return CVVAE_OK;
  int tiles_x, chunks_y;
  const long long grid0 = met_grid(T, H, W, &tiles_x, &chunks_y);
  CVVAE_CHECK_ARG(grid0 < (1ll << 31),   // level 0 has the largest grid
                  "cvvae_frame_ms_ssim: too many frames for one launch (T=%d at %d x %d)", (int)T, (int)H, (int)W);
  const MetWeights wt = met_weights();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  unsigned long long* out = reinterpret_cast<unsigned long long*>(acc);
  CVVAE_CUDA(cudaMemsetAsync(acc, 0, sizeof(int64_t) * kMsLevels * 6 * T, stream));

  frame_metrics_kernel<uint8_t, true><<<static_cast<unsigned>(grid0), kMetThreads, 0, stream>>>(
      a_thwc, b_thwc, H, 3 * W, tiles_x, chunks_y, 3ll * T * H * W, wt, out, 128, 6.5025f, 58.5225f, nullptr);
  CVVAE_LAUNCH_CHECK();
  // levels 1-4 of a, then of b, ...: a_1 | b_1 | a_2 | b_2 | ...
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const void* prev_a = a_thwc;
  const void* prev_b = b_thwc;
  for (int j = 1; j < kMsLevels; ++j) {
    const int Hs = ms_extent(H, j - 1), Ws = ms_extent(W, j - 1), Hd = ms_extent(H, j), Wd = ms_extent(W, j);
    uint16_t* la = reinterpret_cast<uint16_t*>(ws);
    uint16_t* lb = reinterpret_cast<uint16_t*>(ws + ms_level_bytes(T, H, W, j));
    ws += 2 * ms_level_bytes(T, H, W, j);
    const dim3 pool_grid((Hd * Wd * 3 + 255) / 256, static_cast<unsigned>(T < 65535 ? T : 65535), 2);
    if (j == 1)
      ms_pool_kernel<uint8_t><<<pool_grid, 256, 0, stream>>>(a_thwc, b_thwc, la, lb, T, Hs, Ws, Hd, Wd);
    else
      ms_pool_kernel<uint16_t><<<pool_grid, 256, 0, stream>>>(static_cast<const uint16_t*>(prev_a),
                                                              static_cast<const uint16_t*>(prev_b), la, lb, T, Hs, Ws, Hd, Wd);
    CVVAE_LAUNCH_CHECK();
    const float scale = static_cast<float>(1 << (4 * j));   // 16^j: C1 and C2 in units of level-j sums squared
    const long long grid = met_grid(T, Hd, Wd, &tiles_x, &chunks_y);
    frame_metrics_kernel<uint16_t, true><<<static_cast<unsigned>(grid), kMetThreads, 0, stream>>>(
        la, lb, Hd, 3 * Wd, tiles_x, chunks_y, 6ll * T * Hd * Wd, wt, out + 6 * j, 128 << (2 * j), 6.5025f * scale,
        58.5225f * scale, nullptr);
    CVVAE_LAUNCH_CHECK();
    prev_a = la;
    prev_b = lb;
  }
  return CVVAE_OK;
}
