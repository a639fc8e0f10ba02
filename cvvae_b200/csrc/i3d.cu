// FVD's network (Unterthiner et al. 2018): the Kinetics-400 I3D of the widely used PyTorch port (InceptionI3d), in fp32
// with TF32 products.  Its 57 BN-folded convolutions run on the tensor-core convolution (conv_tc, ReLU in the epilogue,
// each Inception branch writing straight into its channel slice of the block's output); this file holds the kernels
// around them:
//
//   i3d_stem_input_kernel: the fp32 channels-first clip [N, 3, T, H, W] (frames_to_training_input's output) -> the input of
//     Conv3d_1a_7x7 (7 x 7 x 7, stride 2, TF "SAME" zero padding) with its 7 x 7 spatial taps of three consecutive frames
//     packed into channels: [N, TP, OH, OW, 448], TP = ceil(T / 2) + 2, OH = ceil(H / 2), OW = ceil(W / 2).  Channel
//     ((j * 7 + kh) * 7 + kw) * 3 + c of (u, oh, ow) is x(c, 2u - ft + j, 2 oh - fh + kh, 2 ow - fw + kw) for j < 3 (ft, fh,
//     fw the front paddings), 0 outside the clip and in channels 441..447, rounded to the nearest TF32 value.  Frame
//     2 t - ft + kt (kt = 2k + j) of output t is then in position t + k, so the stem runs on conv_tc as a 3 x 1 x 1
//     stride-1 convolution whose tap k carries the temporal taps 2k + j (k = 0: kt 0..2; k = 1, 2: j = 1, 2, kt 3..6).
//     conv_tc takes temporal extents up to 3, so the seven taps cannot be left to it one frame per position.
//   i3d_max_pool3d_kernel: 3-D max pool of a channels-last tensor with TF "SAME" zero padding, any (k, s) per axis.
//   i3d_head_kernel: per clip, the [2, 7, 7] average pool of Mixed_5c, the logits (1 x 1 x 1 conv with bias) and the mean
//     over the remaining temporal positions, fp64, one CTA per clip.
#include <math.h>

#include "common.cuh"

namespace cvvae {

constexpr int kI3dThreads = 256;
constexpr int kI3dStemTaps = 3 * 49 * 3;   // three frames x 7 x 7 taps x 3 channels
constexpr int kI3dStemChannels = 448;      // padded to a multiple of 8 channels (conv_tc's channel granularity)
constexpr int kI3dHeadThreads = 512;

// TF "SAME" padding of one axis: the front padding; the output extent is ceil(n / s)
inline int i3d_same_front(int n, int k, int s) {
  const int r = n % s;
  const int pad = r == 0 ? (k - s > 0 ? k - s : 0) : (k - r > 0 ? k - r : 0);
  return pad / 2;
}

// One thread per four channels of a packed position; clips along y, 64-bit offsets across clips, 32-bit within one.
__global__ void __launch_bounds__(kI3dThreads)
    i3d_stem_input_kernel(const float* __restrict__ x, int N, int T, int H, int W, int TP, int OH, int OW, int ft, int fh, int fw,
                          float* __restrict__ out) {
  constexpr int kQ = kI3dStemChannels / 4;
  const int n = TP * OH * OW * kQ;
  const int i = blockIdx.x * kI3dThreads + threadIdx.x;
  if (i >= n) return;
  const int q = i % kQ, pos = i / kQ;
  const int ow = pos % OW, r = pos / OW;
  const int oh = r % OH, u = r / OH;
  const long long plane = static_cast<long long>(H) * W;
  for (int clip = blockIdx.y; clip < N; clip += gridDim.y) {
    const float* src = x + static_cast<long long>(clip) * 3 * T * plane;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ch = 4 * q + e;
      const int j = ch / 147, rem = ch % 147;
      const int kh = rem / 21, kw = (rem / 3) % 7, c = rem % 3;
      const int t = 2 * u - ft + j, y = 2 * oh - fh + kh, xw = 2 * ow - fw + kw;
      const bool in = ch < kI3dStemTaps && t >= 0 && t < T && y >= 0 && y < H && xw >= 0 && xw < W;
      v[e] = in ? tf32_rn(__ldg(src + (static_cast<long long>(c) * T + t) * plane + static_cast<long long>(y) * W + xw)) : 0.f;
    }
    reinterpret_cast<float4*>(out + static_cast<long long>(clip) * n * 4)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

struct I3dPool {
  int k[3], s[3], f[3];   // kernel, stride and front padding per axis (t, h, w)
};

// f [N, T, H, W, C] -> out [N, OT, OH, OW, C]: the maximum over the window, a tap outside the input counting as 0 (zero
// padding, as F.pad followed by F.max_pool3d).  Exact: no rounding (the inputs are ReLU outputs already stored at TF32
// precision where a convolution reads them, and rounding is monotonic).  One thread per four channels of an output
// position, clips along y.
__global__ void __launch_bounds__(kI3dThreads)
    i3d_max_pool3d_kernel(const float* __restrict__ f, int N, int T, int H, int W, int C, int OT, int OH, int OW, I3dPool p,
                          float* __restrict__ out) {
  const int cq = C / 4;
  const int n = OT * OH * OW * cq;
  const int i = blockIdx.x * kI3dThreads + threadIdx.x;
  if (i >= n) return;
  const int q = i % cq, pos = i / cq;
  const int ow = pos % OW, r = pos / OW;
  const int oh = r % OH, ot = r / OH;
  const int t0 = ot * p.s[0] - p.f[0], h0 = oh * p.s[1] - p.f[1], w0 = ow * p.s[2] - p.f[2];
  for (int clip = blockIdx.y; clip < N; clip += gridDim.y) {
    const float4* src = reinterpret_cast<const float4*>(f + static_cast<long long>(clip) * T * H * W * C) + q;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    bool padded = false;
    for (int kt = 0; kt < p.k[0]; ++kt) {
      const int t = t0 + kt;
      for (int kh = 0; kh < p.k[1]; ++kh) {
        const int h = h0 + kh;
        for (int kw = 0; kw < p.k[2]; ++kw) {
          const int w = w0 + kw;
          if (t < 0 || t >= T || h < 0 || h >= H || w < 0 || w >= W) {
            padded = true;
            continue;
          }
          const float4 v = __ldg(src + ((static_cast<long long>(t) * H + h) * W + w) * cq);
          m = make_float4(fmaxf(m.x, v.x), fmaxf(m.y, v.y), fmaxf(m.z, v.z), fmaxf(m.w, v.w));
        }
      }
    }
    if (padded) m = make_float4(fmaxf(m.x, 0.f), fmaxf(m.y, 0.f), fmaxf(m.z, 0.f), fmaxf(m.w, 0.f));
    reinterpret_cast<float4*>(out + static_cast<long long>(clip) * n * 4)[i] = m;
  }
}

// One CTA per clip.  f [N, T, 7, 7, C] fp32 (Mixed_5c), w fp32 [K, C], bias fp32 [K], out fp64 [N, K]:
//   m[c] = mean over p < T - 1 of the mean over (t, h, w) in [p, p + 2) x 7 x 7 of f(t, h, w, c)
//        = sum_t n_t S_t[c] / (98 (T - 1)),  S_t[c] = sum over (h, w) of f(t, h, w, c),  n_t = [t >= 1] + [t < T - 1]
//   out[k] = bias[k] + sum_c w[k][c] m[c]
// (the logits are linear, so the mean over positions of the logits is the logits of the mean), all in fp64.  A thread
// sums its channels over the positions in a fixed order, a warp forms each logit with a fixed-order shuffle reduction:
// the result depends on the clip alone.
__global__ void __launch_bounds__(kI3dHeadThreads)
    i3d_head_kernel(const float* __restrict__ f, int T, int C, const float* __restrict__ w, const float* __restrict__ bias, int K,
                    double* __restrict__ out) {
  extern __shared__ double s_m[];   // [C]
  const int clip = blockIdx.x;
  const float* src = f + static_cast<long long>(clip) * T * 49 * C;
  const double scale = 1.0 / (98.0 * (T - 1));
  for (int c = threadIdx.x; c < C; c += kI3dHeadThreads) {
    double acc = 0.0;
    for (int t = 0; t < T; ++t) {
      double s = 0.0;
      for (int hw = 0; hw < 49; ++hw) s += static_cast<double>(__ldg(src + (static_cast<long long>(t) * 49 + hw) * C + c));
      acc += static_cast<double>((t >= 1) + (t < T - 1)) * s;
    }
    s_m[c] = acc * scale;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < K; k += kI3dHeadThreads / 32) {
    const float* wk = w + static_cast<long long>(k) * C;
    double s = 0.0;
    for (int c = lane; c < C; c += 32) s = fma(static_cast<double>(__ldg(wk + c)), s_m[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[static_cast<long long>(clip) * K + k] = static_cast<double>(bias[k]) + s;
  }
}

// y extent of the grids: clips are walked along y, 32-bit indices within a clip along x
inline dim3 i3d_clip_grid(long long per_clip, long long clips) {
  return dim3(static_cast<unsigned>((per_clip + kI3dThreads - 1) / kI3dThreads),
              static_cast<unsigned>(clips < 65535 ? clips : 65535));
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_i3d_stem_input(const float* x, int32_t N, int32_t T, int32_t H, int32_t W, float* out, void* stream) {
  CVVAE_CHECK_ARG(x && out, "cvvae_i3d_stem_input: null pointer");
  CVVAE_CHECK_ARG(N >= 0 && T >= 1 && H >= 1 && W >= 1, "cvvae_i3d_stem_input: needs N >= 0 and T, H, W >= 1, got N=%d T=%d H=%d W=%d",
                  (int)N, (int)T, (int)H, (int)W);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(x) % sizeof(float) == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                  "cvvae_i3d_stem_input: x must be 4-byte and out 16-byte aligned");
  const int TP = (T + 1) / 2 + 2, OH = (H + 1) / 2, OW = (W + 1) / 2;
  const long long per_clip = 1ll * TP * OH * OW * (kI3dStemChannels / 4);
  CVVAE_CHECK_ARG(per_clip < (1ll << 31) && 3ll * T * H * W < (1ll << 40),
                  "cvvae_i3d_stem_input: a %d x %d x %d clip is too large for one launch", (int)T, (int)H, (int)W);
  if (N == 0) return CVVAE_OK;
  const int ft = i3d_same_front(T, 7, 2), fh = i3d_same_front(H, 7, 2), fw = i3d_same_front(W, 7, 2);
  i3d_stem_input_kernel<<<i3d_clip_grid(per_clip, N), kI3dThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, N, T, H, W, TP, OH, OW, ft, fh, fw, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_i3d_max_pool3d(const float* f, int32_t N, int32_t T, int32_t H, int32_t W, int32_t C, const int32_t* kernel,
                                    const int32_t* stride, float* out, void* stream) {
  CVVAE_CHECK_ARG(f && out && kernel && stride, "cvvae_i3d_max_pool3d: null pointer");
  CVVAE_CHECK_ARG(N >= 0 && T >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0,
                  "cvvae_i3d_max_pool3d: needs N >= 0, T, H, W >= 1 and C a positive multiple of 4, got N=%d T=%d H=%d W=%d C=%d",
                  (int)N, (int)T, (int)H, (int)W, (int)C);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(f) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                  "cvvae_i3d_max_pool3d: f and out must be 16-byte aligned");
  I3dPool p;
  const int n[3] = {T, H, W};
  int o[3];
  for (int a = 0; a < 3; ++a) {
    CVVAE_CHECK_ARG(kernel[a] >= 1 && kernel[a] <= 7 && stride[a] >= 1 && stride[a] <= 7,
                    "cvvae_i3d_max_pool3d: kernel and stride must be 1..7 per axis, got k=%d s=%d on axis %d", (int)kernel[a],
                    (int)stride[a], a);
    p.k[a] = kernel[a];
    p.s[a] = stride[a];
    p.f[a] = i3d_same_front(n[a], kernel[a], stride[a]);
    o[a] = (n[a] + stride[a] - 1) / stride[a];
  }
  CVVAE_CHECK_ARG(1ll * T * H * W * C < (1ll << 31), "cvvae_i3d_max_pool3d: %d x %d x %d x %d is too large for one launch", (int)T,
                  (int)H, (int)W, (int)C);
  if (N == 0) return CVVAE_OK;
  i3d_max_pool3d_kernel<<<i3d_clip_grid(1ll * o[0] * o[1] * o[2] * (C / 4), N), kI3dThreads, 0,
                          static_cast<cudaStream_t>(stream)>>>(f, N, T, H, W, C, o[0], o[1], o[2], p, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_i3d_head(const float* f, int32_t N, int32_t T, int32_t H, int32_t W, int32_t C, const float* w,
                              const float* bias, int32_t K, double* out, void* stream) {
  CVVAE_CHECK_ARG(f && w && bias && out, "cvvae_i3d_head: null pointer");
  CVVAE_CHECK_ARG(N >= 0 && T >= 2 && H == 7 && W == 7,
                  "cvvae_i3d_head: the [2, 7, 7] average pool needs N >= 0, T >= 2 and H = W = 7, got N=%d T=%d H=%d W=%d", (int)N,
                  (int)T, (int)H, (int)W);
  CVVAE_CHECK_ARG(C >= 1 && C <= 4096 && K >= 1, "cvvae_i3d_head: needs 1 <= C <= 4096 and K >= 1, got C=%d K=%d", (int)C,
                  (int)K);
  CVVAE_CHECK_ARG(reinterpret_cast<uintptr_t>(f) % sizeof(float) == 0 && reinterpret_cast<uintptr_t>(w) % sizeof(float) == 0 &&
                      reinterpret_cast<uintptr_t>(bias) % sizeof(float) == 0 &&
                      reinterpret_cast<uintptr_t>(out) % sizeof(double) == 0,
                  "cvvae_i3d_head: f, w and bias must be 4-byte and out 8-byte aligned");
  if (N == 0) return CVVAE_OK;
  i3d_head_kernel<<<static_cast<unsigned>(N), kI3dHeadThreads, C * sizeof(double), static_cast<cudaStream_t>(stream)>>>(
      f, T, C, w, bias, K, out);
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
