// LPIPS (Zhang et al. 2018, VGG16 variant) of two uint8 videos, the learned perceptual distance the reference adds to its
// reconstruction loss per frame (lvdm/modules/autoencoding/losses/discriminator_loss.py:239-256,
// lvdm/modules/autoencoding/lpips/loss/lpips.py).  The thirteen 3 x 3 convolutions run on the tensor-core convolution
// (conv_tc, fp32 activations, TF32 products, ReLU in its epilogue); this file holds the two kernels around them:
//
//   lpips_input_kernel: uint8 frames of both videos -> the scaled input of conv1_1 with its nine spatial taps packed
//     into 32 channels, so that conv1_1 runs as a 1 x 1 convolution (as the engine runs conv_in).  A CTA first builds
//     the 3 x 256 table of scaled byte values, which are all the values the input can take.
//   lpips_tap_kernel: one tap (relu1_2 .. relu5_3) of both videos -> per frame, the sum over positions of
//     sum_c w[c] (f_a / (|f_a| + eps) - f_b / (|f_b| + eps))^2, and optionally the 2 x 2 max pool of every image for the
//     next block, in the same pass, rounded to the nearest TF32 value like every input of a convolution here.  One warp
//     scores one position at a time (each lane holds C / 32 channels), walking 2 x 2 quads so that a full quad's pooled
//     maximum is formed in registers on the way.  lpips_tap_copy_kernel is the same pass writing, instead of the pool, a
//     TF32-rounded copy of the tap for a convolution that reads it (AlexNet's relu3 and relu4).
//
// LPIPS on AlexNet features (net='alex') runs its five convolutions on conv_tc too; conv1 (11 x 11, stride 4) and conv2
// (5 x 5) as 1 x 1 convolutions over their taps packed into channels by lpips_alex_input_kernel (from the uint8 frames,
// 384 channels) and lpips_pack5x5_kernel (1600 channels), with lpips_max_pool3s2_kernel for the 3 x 3 stride-2 pools.
//
// LPIPS maps (lpips spatial=True, either network): lpips_tap_map_kernel is the tap pass, with its pool or copy, that also
// keeps every position's weighted difference in an fp64 tap map; lpips_upsample_sum_kernel then upsamples the five tap
// maps bilinearly to the frame and sums them.  The frame sums run exactly as without maps, so the scalar is unchanged.
//
// The normalisation and the difference are fp64: a good reconstruction's f_a / |f_a| - f_b / |f_b| is small next to
// either term, and fp32 would leave a relative error of 1e-7 / |difference| in it.  Accumulation: a warp keeps one
// fp64 partial per lane over its positions, a CTA reduces its warps in a fixed order and adds its sum, rounded once to
// units of 2^-32, to the frame's int64 with an integer atomic.  The CTA -> positions map depends on H and W alone, so a
// frame's result is bit-reproducible and independent of the other frames in the call; identical frames give exactly 0
// and swapping the videos gives the same bits (the expression is symmetric in a and b, term by term).
#include <math.h>

#include "common.cuh"

namespace cvvae {

constexpr int kLpInThreads = 256;
constexpr int kLpInChannels = 32;     // 27 taps x channels, padded to a channel block of fp32 storage
constexpr int kLpTapThreads = 256;
constexpr int kLpQuadsPerWarp = 4;
constexpr int kLpQuadsPerCta = kLpQuadsPerWarp * kLpTapThreads / 32;
constexpr long long kLpMaxPositions = 1ll << 23;   // H * W of one tap: with |w| <= 32 the frame sum stays below 2^62 / 2^32

// (x - shift) / scale of ScalingLayer (lpips.py:67-78), x = byte / 127.5 - 1, each operation one fp32 rounding as PyTorch
// evaluates it, then rounded to the nearest TF32 value: the input's only consumer is a tensor-core product.
__device__ __forceinline__ float lpips_scaled(int byte, int c) {
  const float shift = c == 0 ? -0.030f : c == 1 ? -0.088f : -0.188f;
  const float scale = c == 0 ? 0.458f : c == 1 ? 0.448f : 0.450f;
  const float x = __fsub_rn(__fdiv_rn(static_cast<float>(byte), 127.5f), 1.0f);
  return tf32_rn(__fdiv_rn(__fsub_rn(x, shift), scale));
}

// out [2T, H, W, 32]: image i < T is frame i of a, image T + i frame i of b; channel (kh*3 + kw)*3 + c of position
// (h, w) is the scaled pixel (h + kh - 1, w + kw - 1, c), 0 outside the frame (conv2d pads the scaled input with zeros),
// channels 27..31 are 0.  One thread per output position: 32 floats, eight 16-byte stores.
__global__ void __launch_bounds__(kLpInThreads)
    lpips_input_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int T, int H, int W,
                       float* __restrict__ out) {
  __shared__ float s_tab[3][256];
  for (int i = threadIdx.x; i < 3 * 256; i += kLpInThreads) s_tab[i >> 8][i & 255] = lpips_scaled(i & 255, i >> 8);
  __syncthreads();
  const long long n = 2ll * T * H * W;
  const long long pos = static_cast<long long>(blockIdx.x) * kLpInThreads + threadIdx.x;
  if (pos >= n) return;
  const int w = static_cast<int>(pos % W);
  const long long r = pos / W;
  const int h = static_cast<int>(r % H);
  const int img = static_cast<int>(r / H);
  const uint8_t* src = (img < T ? a + static_cast<long long>(img) * H * W * 3 : b + static_cast<long long>(img - T) * H * W * 3);
  float v[kLpInChannels];
#pragma unroll
  for (int kh = 0; kh < 3; ++kh)
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int y = h + kh - 1, x = w + kw - 1;
      const bool in = y >= 0 && y < H && x >= 0 && x < W;
      const uint8_t* px = src + (static_cast<long long>(y) * W + x) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) v[(kh * 3 + kw) * 3 + c] = in ? s_tab[c][px[c]] : 0.f;
    }
#pragma unroll
  for (int c = 27; c < kLpInChannels; ++c) v[c] = 0.f;
  float4* dst = reinterpret_cast<float4*>(out + pos * kLpInChannels);
#pragma unroll
  for (int i = 0; i < kLpInChannels / 4; ++i) dst[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}

// AlexNet's conv1 (11 x 11, stride 4, zero padding 2, lpips net='alex') as a 1 x 1 convolution over its 3 * 11 * 11 = 363
// taps, padded to 384 channels.  out [2T, OH, OW, 384], OH = (H - 7) / 4 + 1 (likewise OW): channel (c * 11 + kh) * 11 + kw
// of position (oh, ow) is the scaled pixel (4 oh + kh - 2, 4 ow + kw - 2, c) as lpips_input_kernel computes it, 0 outside
// the frame and in channels 363..383; the channel order is that of the PyTorch weight [64, 3, 11, 11] flattened.  One
// thread per four channels of a position (one 16-byte store), so consecutive threads write consecutive bytes.  The index
// within an image is 32-bit (the entry point checks OH * OW * 96 < 2^31), images are walked along y with 64-bit offsets.
constexpr int kLpAlexK = 11;
constexpr int kLpAlexTaps = 3 * kLpAlexK * kLpAlexK;
constexpr int kLpAlexInChannels = 384;
__global__ void __launch_bounds__(kLpInThreads)
    lpips_alex_input_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int T, int H, int W, int OH, int OW,
                            float* __restrict__ out) {
  __shared__ float s_tab[3][256];
  for (int i = threadIdx.x; i < 3 * 256; i += kLpInThreads) s_tab[i >> 8][i & 255] = lpips_scaled(i & 255, i >> 8);
  __syncthreads();
  constexpr int kQ = kLpAlexInChannels / 4;
  const int n = OH * OW * kQ;
  const int i = blockIdx.x * kLpInThreads + threadIdx.x;
  if (i >= n) return;
  const int q = i % kQ, pos = i / kQ;
  const int oh = pos / OW, ow = pos % OW;
  for (int img = blockIdx.y; img < 2 * T; img += gridDim.y) {
    const uint8_t* src = img < T ? a + static_cast<long long>(img) * H * W * 3 : b + static_cast<long long>(img - T) * H * W * 3;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ch = 4 * q + j;
      const int c = ch / (kLpAlexK * kLpAlexK), k = ch % (kLpAlexK * kLpAlexK);
      const int y = 4 * oh + k / kLpAlexK - 2, x = 4 * ow + k % kLpAlexK - 2;
      const bool in = ch < kLpAlexTaps && y >= 0 && y < H && x >= 0 && x < W;
      v[j] = in ? s_tab[c][src[(static_cast<long long>(y) * W + x) * 3 + c]] : 0.f;
    }
    reinterpret_cast<float4*>(out + static_cast<long long>(img) * n * 4)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// 3 x 3 max pool, stride 2, no padding, floor (AlexNet's features[2] and [5]): out [N, OH, OW, C], OH = (H - 3) / 2 + 1, of
// f [N, H, W, C], rounded to the nearest TF32 value (its only consumer is a convolution; rounding is monotonic, so this is
// the pool of the rounded values).  One thread per four channels of an output position.
__global__ void __launch_bounds__(kLpInThreads)
    lpips_max_pool3s2_kernel(const float* __restrict__ f, int N, int H, int W, int C, int OH, int OW, float* __restrict__ out) {
  const int cq = C / 4;
  const int n = OH * OW * cq;
  const int i = blockIdx.x * kLpInThreads + threadIdx.x;
  if (i >= n) return;
  const int q = i % cq, pos = i / cq;
  const int oh = pos / OW, ow = pos % OW;
  for (int img = blockIdx.y; img < N; img += gridDim.y) {
    const float4* src = reinterpret_cast<const float4*>(f + static_cast<long long>(img) * H * W * C) + q;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const float4 v = __ldg(src + (static_cast<long long>(2 * oh + kh) * W + 2 * ow + kw) * cq);
        m = make_float4(fmaxf(m.x, v.x), fmaxf(m.y, v.y), fmaxf(m.z, v.z), fmaxf(m.w, v.w));
      }
    reinterpret_cast<float4*>(out + static_cast<long long>(img) * n * 4)[i] =
        make_float4(tf32_rn(m.x), tf32_rn(m.y), tf32_rn(m.z), tf32_rn(m.w));
  }
}

// The 5 x 5 taps (zero padding 2) of x [N, H, W, C] packed into channels, so that AlexNet's conv2 runs as a 1 x 1
// convolution: out [N, H, W, 25 C], channel (kh * 5 + kw) * C + c of position (h, w) is x(h + kh - 2, w + kw - 2, c), 0
// outside the image.  An exact copy.  One thread per four channels of an output position.
__global__ void __launch_bounds__(kLpInThreads)
    lpips_pack5x5_kernel(const float* __restrict__ x, int N, int H, int W, int C, float* __restrict__ out) {
  const int cq = C / 4, oq = 25 * cq;
  const int n = H * W * oq;
  const int i = blockIdx.x * kLpInThreads + threadIdx.x;
  if (i >= n) return;
  const int q = i % oq, pos = i / oq;
  const int tap = q / cq, c4 = q % cq;
  const int y = pos / W + tap / 5 - 2, xw = pos % W + tap % 5 - 2;
  const bool in = y >= 0 && y < H && xw >= 0 && xw < W;
  for (int img = blockIdx.y; img < N; img += gridDim.y) {
    const float4* src = reinterpret_cast<const float4*>(x + static_cast<long long>(img) * H * W * C);
    reinterpret_cast<float4*>(out + static_cast<long long>(img) * n * 4)[i] =
        in ? __ldg(src + (static_cast<long long>(y) * W + xw) * cq + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// kV consecutive channels of one position, lane l holding [l*kV, l*kV + kV)
template <int kV>
__device__ __forceinline__ void lp_load(const float* p, float (&v)[kV]) {
  if constexpr (kV == 2) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(p));
    v[0] = q.x;
    v[1] = q.y;
  } else if constexpr (kV % 4 == 2) {   // C = 192: 24 bytes per lane, 8-byte aligned
#pragma unroll
    for (int i = 0; i < kV / 2; ++i) {
      const float2 q = __ldg(reinterpret_cast<const float2*>(p) + i);
      v[2 * i] = q.x;
      v[2 * i + 1] = q.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < kV / 4; ++i) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(p) + i);
      v[4 * i] = q.x;
      v[4 * i + 1] = q.y;
      v[4 * i + 2] = q.z;
      v[4 * i + 3] = q.w;
    }
  }
}
template <int kV>
__device__ __forceinline__ void lp_store(float* p, const float (&v)[kV]) {
  if constexpr (kV == 2) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  } else if constexpr (kV % 4 == 2) {
#pragma unroll
    for (int i = 0; i < kV / 2; ++i) reinterpret_cast<float2*>(p)[i] = make_float2(v[2 * i], v[2 * i + 1]);
  } else {
#pragma unroll
    for (int i = 0; i < kV / 4; ++i)
      reinterpret_cast<float4*>(p)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// f [2T, H, W, C] (frames of a, then of b); acc[t] += sum over the frame's positions of the weighted squared difference
// of the normalised features, in units of 2^-32.  pooled (optional) [2T, H/2, W/2, C]: 2 x 2 max pool, floor, rounded to
// TF32 (rounding is monotonic, so this is the rounded max of the four values).
// CTA (t, blk) owns quads [blk * 32, blk * 32 + 32) of frame t in row-major quad order; warp w of it quads 4w .. 4w + 3.
// kCopy: `pooled` is instead `copy` [2T, H, W, C], which receives every position of f rounded to the nearest TF32 value
// (a tap whose next consumer is a convolution, AlexNet's relu3 and relu4); there is no pool.
// kMap: also map [T, H, W] (fp64) = each position's weighted squared difference, summed in its own fp64 accumulator (the
// lane's channels, then the warp) and stored by lane 0; `part`, the frame sum's accumulator, runs exactly as without it.
// The map is exactly 0 where the features agree and the same bits with a and b swapped.
template <int C, bool kCopy, bool kMap = false>
__device__ __forceinline__ void lpips_tap(const float* __restrict__ f, int T, int H, int W, const float* __restrict__ lin_w,
                                          unsigned long long* __restrict__ acc, float* __restrict__ pooled, int ctas_per_frame,
                                          double* __restrict__ map = nullptr) {
  constexpr int kV = C / 32;
  __shared__ double s_red[kLpTapThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x / ctas_per_frame, blk = blockIdx.x % ctas_per_frame;
  const int QW = (W + 1) / 2, QH = (H + 1) / 2, PH = H / 2, PW = W / 2;
  const long long img_stride = static_cast<long long>(H) * W * C;
  const float* fa = f + static_cast<long long>(t) * img_stride + lane * kV;
  const float* fb = f + static_cast<long long>(T + t) * img_stride + lane * kV;
  double wc[kV];
  {
    float wf[kV];
    lp_load<kV>(lin_w + lane * kV, wf);
#pragma unroll
    for (int i = 0; i < kV; ++i) wc[i] = wf[i];
  }
  double part = 0.0;
  for (int i = 0; i < kLpQuadsPerWarp; ++i) {
    const long long q = static_cast<long long>(blk) * kLpQuadsPerCta + warp * kLpQuadsPerWarp + i;
    if (q >= static_cast<long long>(QH) * QW) break;   // warp-uniform
    const int qh = static_cast<int>(q / QW), qw = static_cast<int>(q % QW);
    const bool full = qh < PH && qw < PW;
    float ma[kV], mb[kV];
#pragma unroll
    for (int k = 0; k < kV; ++k) ma[k] = mb[k] = -INFINITY;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int h = 2 * qh + (p >> 1), w = 2 * qw + (p & 1);
      if (h >= H || w >= W) continue;   // warp-uniform: the last row / column of an odd extent
      const long long off = (static_cast<long long>(h) * W + w) * C;
      float va[kV], vb[kV];
      lp_load<kV>(fa + off, va);
      lp_load<kV>(fb + off, vb);
      if constexpr (kCopy) {
        float ra[kV], rb[kV];
#pragma unroll
        for (int k = 0; k < kV; ++k) {
          ra[k] = tf32_rn(va[k]);
          rb[k] = tf32_rn(vb[k]);
        }
        lp_store<kV>(pooled + (fa - f) + off, ra);
        lp_store<kV>(pooled + (fb - f) + off, rb);
      }
      double sa = 0.0, sb = 0.0;
#pragma unroll
      for (int k = 0; k < kV; ++k) {
        sa = fma(static_cast<double>(va[k]), static_cast<double>(va[k]), sa);
        sb = fma(static_cast<double>(vb[k]), static_cast<double>(vb[k]), sb);
      }
      sa = warp_sum(sa);
      sb = warp_sum(sb);
      // f / (sqrt(sum f^2 + 1e-10) + 1e-10), lpips.py:141-143, as a product with the reciprocal
      const double ra = 1.0 / (sqrt(sa + 1e-10) + 1e-10), rb = 1.0 / (sqrt(sb + 1e-10) + 1e-10);
      double pos = 0.0;
#pragma unroll
      for (int k = 0; k < kV; ++k) {
        const double d = static_cast<double>(va[k]) * ra - static_cast<double>(vb[k]) * rb;
        part = fma(wc[k], d * d, part);
        if constexpr (kMap) {
          // d again with explicit roundings: the compiler may fuse d's product and difference into one FMA, which leaves
          // the rounding error of the other product (about 1e-17) where a and b agree.  The frame sum rounds that away,
          // a map would show it; this d is exactly 0 for equal features and exactly -d with a and b swapped.
          const double dm = __dsub_rn(__dmul_rn(static_cast<double>(va[k]), ra), __dmul_rn(static_cast<double>(vb[k]), rb));
          pos = fma(wc[k], dm * dm, pos);
        }
        ma[k] = fmaxf(ma[k], va[k]);
        mb[k] = fmaxf(mb[k], vb[k]);
      }
      if constexpr (kMap) {
        pos = warp_sum(pos);
        if (lane == 0) map[(static_cast<long long>(t) * H + h) * W + w] = pos;
      }
    }
    if (!kCopy && pooled && full) {
      const long long po = (static_cast<long long>(qh) * PW + qw) * C + lane * kV;
      const long long pstride = static_cast<long long>(PH) * PW * C;
#pragma unroll
      for (int k = 0; k < kV; ++k) {
        ma[k] = tf32_rn(ma[k]);
        mb[k] = tf32_rn(mb[k]);
      }
      lp_store<kV>(pooled + static_cast<long long>(t) * pstride + po, ma);
      lp_store<kV>(pooled + static_cast<long long>(T + t) * pstride + po, mb);
    }
  }
  part = warp_sum(part);
  if (lane == 0) s_red[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < kLpTapThreads / 32; ++i) s += s_red[i];
    atomicAdd(acc + t, static_cast<unsigned long long>(__double2ll_rn(s * 4294967296.0)));
  }
}

// Two CTAs per SM at least below C = 384: left to itself ptxas gives C = 64 / 128 48 / 64 registers and spills.
template <int C>
__global__ void __launch_bounds__(kLpTapThreads, C >= 384 ? 1 : 2)
    lpips_tap_kernel(const float* __restrict__ f, int T, int H, int W, const float* __restrict__ lin_w,
                     unsigned long long* __restrict__ acc, float* __restrict__ pooled, int ctas_per_frame) {
  lpips_tap<C, false>(f, T, H, W, lin_w, acc, pooled, ctas_per_frame);
}
template <int C>
__global__ void __launch_bounds__(kLpTapThreads, C >= 384 ? 1 : 2)
    lpips_tap_copy_kernel(const float* __restrict__ f, int T, int H, int W, const float* __restrict__ lin_w,
                          unsigned long long* __restrict__ acc, float* __restrict__ copy, int ctas_per_frame) {
  lpips_tap<C, true>(f, T, H, W, lin_w, acc, copy, ctas_per_frame);
}
// either of the above (kCopy: `side` is `copy`, else `pooled`) that also writes the tap's map
template <int C, bool kCopy>
__global__ void __launch_bounds__(kLpTapThreads, C >= 384 ? 1 : 2)
    lpips_tap_map_kernel(const float* __restrict__ f, int T, int H, int W, const float* __restrict__ lin_w,
                         unsigned long long* __restrict__ acc, float* __restrict__ side, int ctas_per_frame,
                         double* __restrict__ map) {
  lpips_tap<C, kCopy, true>(f, T, H, W, lin_w, acc, side, ctas_per_frame, map);
}

// One tap kernel of the family the entry point selects: plain, with the TF32 copy, or (kMap) either one with the map.
template <int C, bool kCopy, bool kMap>
void lpips_tap_kernel_launch(unsigned grid, cudaStream_t stream, const float* f, int T, int H, int W, const float* lin_w,
                             unsigned long long* acc, float* side, int ctas_per_frame, double* map) {
  if constexpr (kMap)
    lpips_tap_map_kernel<C, kCopy><<<grid, kLpTapThreads, 0, stream>>>(f, T, H, W, lin_w, acc, side, ctas_per_frame, map);
  else if constexpr (kCopy)
    lpips_tap_copy_kernel<C><<<grid, kLpTapThreads, 0, stream>>>(f, T, H, W, lin_w, acc, side, ctas_per_frame);
  else
    lpips_tap_kernel<C><<<grid, kLpTapThreads, 0, stream>>>(f, T, H, W, lin_w, acc, side, ctas_per_frame);
}

// The taps' maps upsampled to the frame and summed, lpips' spatial=True: out [T, H, W] fp32 = sum over k of the bilinear
// upsampling (align_corners=False) of tap map k, maps [T, h_k, w_k] fp64 back to back in `taps` from offset off[k].
// Source positions follow PyTorch's rule for fp32 tensors (scale = in / out, src = max(scale (dst + 0.5) - 0.5, 0), each
// an fp32 rounding; i0 = floor, i1 = i0 + 1 clamped to in - 1, lambda = src - i0); the interpolation and the sum are fp64,
// rounded to fp32 once.  One thread per output pixel.
constexpr int kLpMaps = 5;
constexpr int kLpUpThreads = 256;
struct LpTapMaps {
  int h[kLpMaps], w[kLpMaps];
  long long off[kLpMaps];
};

__device__ __forceinline__ void lp_source(int dst, int in, int out, int& i0, int& i1, double& lambda) {
  const float scale = __fdiv_rn(static_cast<float>(in), static_cast<float>(out));
  const float src = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn(static_cast<float>(dst), 0.5f)), 0.5f), 0.f);
  i0 = static_cast<int>(src);
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  lambda = static_cast<double>(__fsub_rn(src, static_cast<float>(i0)));
}

__global__ void __launch_bounds__(kLpUpThreads)
    lpips_upsample_sum_kernel(const double* __restrict__ taps, int H, int W, long long n, LpTapMaps m, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * kLpUpThreads + threadIdx.x;
  if (i >= n) return;
  const int x = static_cast<int>(i % W);
  const long long r = i / W;
  const int y = static_cast<int>(r % H);
  const long long t = r / H;
  double sum = 0.0;
#pragma unroll
  for (int k = 0; k < kLpMaps; ++k) {
    int y0, y1, x0, x1;
    double ly, lx;
    lp_source(y, m.h[k], H, y0, y1, ly);
    lp_source(x, m.w[k], W, x0, x1, lx);
    const double* p = taps + m.off[k] + t * m.h[k] * m.w[k];
    const double* p0 = p + static_cast<long long>(y0) * m.w[k];
    const double* p1 = p + static_cast<long long>(y1) * m.w[k];
    const double top = (1.0 - lx) * __ldg(p0 + x0) + lx * __ldg(p0 + x1);
    const double bot = (1.0 - lx) * __ldg(p1 + x0) + lx * __ldg(p1 + x1);
    sum += (1.0 - ly) * top + ly * bot;
  }
  out[i] = static_cast<float>(sum);
}

// y extent of the pixel kernels' grids: images are walked along y, 32-bit indices within an image along x
inline dim3 lp_image_grid(int per_image, long long images) {
  return dim3(static_cast<unsigned>((per_image + kLpInThreads - 1) / kLpInThreads),
              static_cast<unsigned>(images < 65535 ? images : 65535));
}

// the checks and launch shared by cvvae_lpips_tap (pooled: NULL or the 2 x 2 pool), cvvae_lpips_tap_copy and, with kMap,
// cvvae_lpips_tap_map (map required)
template <bool kCopy, bool kMap = false>
int lpips_tap_launch(const char* who, const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w,
                     int64_t* acc, float* pooled, void* stream_, double* map = nullptr) {
  const char* side = kCopy ? "copy" : "pooled";
  CVVAE_CHECK_ARG(f && lin_w && acc && (!kCopy || pooled) && (!kMap || map), "%s: null pointer", who);
  if (kMap) CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(map) % sizeof(double) == 0, "%s: `map` must be 8-byte aligned", who);
  if (kCopy)
    CVVAE_CHECK_ARG(C == 256 || C == 384, "%s: C must be 256 or 384, got %d", who, (int)C);
  else
    CVVAE_CHECK_ARG(C == 64 || C == 128 || C == 192 || C == 256 || C == 384 || C == 512,
                    "%s: C must be 64, 128, 192, 256, 384 or 512, got %d", who, (int)C);
  CVVAE_CHECK_ARG(T >= 0 && H >= 1 && W >= 1, "%s: needs T >= 0 and H, W >= 1, got T=%d H=%d W=%d", who, (int)T, (int)H,
                  (int)W);
  CVVAE_CHECK_ARG(kCopy || !pooled || (H >= 2 && W >= 2), "%s: pooling needs H, W >= 2, got %d x %d", who, (int)H, (int)W);
  CVVAE_CHECK_ARG(1ll * H * W <= kLpMaxPositions,
                  "%s: %d x %d positions exceed the 64-bit accumulator's range (H*W <= 2^23)", who, (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(f) % 16 == 0 && reinterpret_cast<uintptr_t>(lin_w) % 16 == 0 &&
                      reinterpret_cast<uintptr_t>(pooled) % 16 == 0,
                  "%s: f, lin_w and %s must be 16-byte aligned", who, side);
  if (T == 0) return CVVAE_OK;
  const long long quads = 1ll * ((H + 1) / 2) * ((W + 1) / 2);
  const long long per_frame = (quads + kLpQuadsPerCta - 1) / kLpQuadsPerCta;
  const long long grid = per_frame * T;
  CVVAE_CHECK_ARG(grid < (1ll << 31), "%s: too many frames for one launch (T=%d at %d x %d)", who, (int)T, (int)H, (int)W);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_CUDA(cudaMemsetAsync(acc, 0, sizeof(int64_t) * T, stream));
  unsigned long long* out = reinterpret_cast<unsigned long long*>(acc);
  const unsigned g = static_cast<unsigned>(grid);
  const int pf = static_cast<int>(per_frame);
  if constexpr (kCopy) {
    if (C == 256) lpips_tap_kernel_launch<256, true, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else lpips_tap_kernel_launch<384, true, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
  } else {
    if (C == 64) lpips_tap_kernel_launch<64, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else if (C == 128) lpips_tap_kernel_launch<128, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else if (C == 192) lpips_tap_kernel_launch<192, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else if (C == 256) lpips_tap_kernel_launch<256, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else if (C == 384) lpips_tap_kernel_launch<384, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
    else lpips_tap_kernel_launch<512, false, kMap>(g, stream, f, T, H, W, lin_w, out, pooled, pf, map);
  }
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_lpips_input(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, float* out,
                                 void* stream) {
  CVVAE_CHECK_ARG(a_thwc && b_thwc && out, "cvvae_lpips_input: null pointer");
  CVVAE_CHECK_ARG(T >= 0 && H >= 1 && W >= 1, "cvvae_lpips_input: needs T >= 0 and H, W >= 1, got T=%d H=%d W=%d", (int)T,
                  (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0, "cvvae_lpips_input: `out` must be 16-byte aligned");
  if (T == 0) return CVVAE_OK;
  const long long grid = (2ll * T * H * W + kLpInThreads - 1) / kLpInThreads;
  CVVAE_CHECK_ARG(grid < (1ll << 31), "cvvae_lpips_input: too many positions for one launch (T=%d at %d x %d)", (int)T,
                  (int)H, (int)W);
  lpips_input_kernel<<<static_cast<unsigned>(grid), kLpInThreads, 0, static_cast<cudaStream_t>(stream)>>>(a_thwc, b_thwc, T,
                                                                                                         H, W, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_lpips_tap(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w, int64_t* acc,
                               float* pooled, void* stream) {
  return lpips_tap_launch<false>("cvvae_lpips_tap", f, T, H, W, C, lin_w, acc, pooled, stream);
}

extern "C" int cvvae_lpips_tap_copy(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w,
                                    int64_t* acc, float* copy, void* stream) {
  return lpips_tap_launch<true>("cvvae_lpips_tap_copy", f, T, H, W, C, lin_w, acc, copy, stream);
}

extern "C" int cvvae_lpips_tap_map(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w,
                                   int64_t* acc, float* pooled, float* copy, double* map, void* stream) {
  CVVAE_CHECK_ARG(!(pooled && copy), "cvvae_lpips_tap_map: at most one of pooled and copy may be set");
  if (copy) return lpips_tap_launch<true, true>("cvvae_lpips_tap_map", f, T, H, W, C, lin_w, acc, copy, stream, map);
  return lpips_tap_launch<false, true>("cvvae_lpips_tap_map", f, T, H, W, C, lin_w, acc, pooled, stream, map);
}

extern "C" int cvvae_lpips_upsample_sum(const double* taps, int32_t T, int32_t H, int32_t W, const int32_t* tap_hw, float* out,
                                        void* stream) {
  CVVAE_CHECK_ARG(taps && tap_hw && out, "cvvae_lpips_upsample_sum: null pointer");
  CVVAE_CHECK_ARG(T >= 0 && H >= 1 && W >= 1 && 1ll * H * W < (1ll << 31),
                  "cvvae_lpips_upsample_sum: needs T >= 0 and 1 <= H * W < 2^31, got T=%d H=%d W=%d", (int)T, (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(taps) % sizeof(double) == 0 && reinterpret_cast<uintptr_t>(out) % sizeof(float) == 0,
                  "cvvae_lpips_upsample_sum: taps must be 8-byte and out 4-byte aligned");
  LpTapMaps m;
  long long off = 0;
  for (int k = 0; k < kLpMaps; ++k) {
    m.h[k] = tap_hw[2 * k];
    m.w[k] = tap_hw[2 * k + 1];
    CVVAE_CHECK_ARG(m.h[k] >= 1 && m.w[k] >= 1 && 1ll * m.h[k] * m.w[k] < (1ll << 31),
                    "cvvae_lpips_upsample_sum: tap %d is %d x %d; needs 1 <= h * w < 2^31", k, (int)m.h[k], (int)m.w[k]);
    m.off[k] = off;
    off += 1ll * T * m.h[k] * m.w[k];
  }
  if (T == 0) return CVVAE_OK;
  const long long n = 1ll * T * H * W;
  const long long grid = (n + kLpUpThreads - 1) / kLpUpThreads;
  CVVAE_CHECK_ARG(grid < (1ll << 31), "cvvae_lpips_upsample_sum: too many positions for one launch (T=%d at %d x %d)", (int)T,
                  (int)H, (int)W);
  lpips_upsample_sum_kernel<<<static_cast<unsigned>(grid), kLpUpThreads, 0, static_cast<cudaStream_t>(stream)>>>(taps, H, W, n,
                                                                                                                 m, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_lpips_alex_input(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, float* out,
                                      void* stream) {
  CVVAE_CHECK_ARG(a_thwc && b_thwc && out, "cvvae_lpips_alex_input: null pointer");
  CVVAE_CHECK_ARG(T >= 0 && H >= 7 && W >= 7, "cvvae_lpips_alex_input: needs T >= 0 and H, W >= 7, got T=%d H=%d W=%d",
                  (int)T, (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0, "cvvae_lpips_alex_input: `out` must be 16-byte aligned");
  const int OH = (H - 7) / 4 + 1, OW = (W - 7) / 4 + 1;
  CVVAE_CHECK_ARG(1ll * OH * OW * (kLpAlexInChannels / 4) < (1ll << 31),
                  "cvvae_lpips_alex_input: %d x %d frames are too large for one launch", (int)H, (int)W);
  if (T == 0) return CVVAE_OK;
  lpips_alex_input_kernel<<<lp_image_grid(OH * OW * (kLpAlexInChannels / 4), 2ll * T), kLpInThreads, 0,
                            static_cast<cudaStream_t>(stream)>>>(a_thwc, b_thwc, T, H, W, OH, OW, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_lpips_max_pool3s2(const float* f, int32_t N, int32_t H, int32_t W, int32_t C, float* out, void* stream) {
  CVVAE_CHECK_ARG(f && out, "cvvae_lpips_max_pool3s2: null pointer");
  CVVAE_CHECK_ARG(N >= 0 && H >= 3 && W >= 3 && C >= 4 && C % 4 == 0,
                  "cvvae_lpips_max_pool3s2: needs N >= 0, H, W >= 3 and C a positive multiple of 4, got N=%d H=%d W=%d C=%d",
                  (int)N, (int)H, (int)W, (int)C);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(f) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                  "cvvae_lpips_max_pool3s2: f and out must be 16-byte aligned");
  const int OH = (H - 3) / 2 + 1, OW = (W - 3) / 2 + 1;
  CVVAE_CHECK_ARG(1ll * H * W * C < (1ll << 31), "cvvae_lpips_max_pool3s2: %d x %d x %d is too large for one launch", (int)H,
                  (int)W, (int)C);
  if (N == 0) return CVVAE_OK;
  lpips_max_pool3s2_kernel<<<lp_image_grid(OH * OW * (C / 4), N), kLpInThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      f, N, H, W, C, OH, OW, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_lpips_pack5x5(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, float* out, void* stream) {
  CVVAE_CHECK_ARG(x && out, "cvvae_lpips_pack5x5: null pointer");
  CVVAE_CHECK_ARG(N >= 0 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0,
                  "cvvae_lpips_pack5x5: needs N >= 0, H, W >= 1 and C a positive multiple of 4, got N=%d H=%d W=%d C=%d",
                  (int)N, (int)H, (int)W, (int)C);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                  "cvvae_lpips_pack5x5: x and out must be 16-byte aligned");
  CVVAE_CHECK_ARG(25ll * H * W * C < (1ll << 31), "cvvae_lpips_pack5x5: %d x %d x %d is too large for one launch", (int)H,
                  (int)W, (int)C);
  if (N == 0) return CVVAE_OK;
  lpips_pack5x5_kernel<<<lp_image_grid(H * W * 25 * (C / 4), N), kLpInThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, N, H, W, C, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
