// Pixel pre/post-processing either side of encode()/decode(), fused into one pass each (SURVEY.md section 8f row 3):
//   uint8 [T,H,W,3] frames  ->  16-bit [1,3,T,H,W] in [-1,1]   (cvvae_inference_video.py:30-38: `.half() / 127.5 - 1.0`)
//   16-bit [1,3,T,H,W]      ->  uint8 [T,H,W,3]                (cvvae_inference_video.py:47-50: clamp, +1, *127.5, uint8)
// Bit-exact with the reference expressions: every intermediate is rounded to the 16-bit type exactly where PyTorch
// rounds it (each elementwise op reads/writes the tensor dtype, arithmetic in fp32).
#include "common.cuh"

namespace cvvae {

template <int DT>
__global__ void __launch_bounds__(256) u8_to_f16_kernel(const uint8_t* __restrict__ in, typename Elem<DT>::T* __restrict__ out,
                                                        long long thw) {
  using E = Elem<DT>;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < thw;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const typename E::T h = E::from_f(static_cast<float>(in[i * 3 + c]));   // .half() (exact for 0..255; bf16 rounds)
      const typename E::T q = E::from_f(E::to_f(h) / 127.5f);                  // / 127.5
      out[c * thw + i] = E::from_f(E::to_f(q) - 1.0f);                         // - 1.0
    }
  }
}

template <int DT>
__global__ void __launch_bounds__(256) f16_to_u8_kernel(const typename Elem<DT>::T* __restrict__ in, uint8_t* __restrict__ out,
                                                        long long thw) {
  using E = Elem<DT>;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < thw;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = E::to_f(in[c * thw + i]);
      v = fminf(fmaxf(v, -1.0f), 1.0f);                 // torch.clamp(x, -1, 1)   (NaN propagates like torch: stays NaN)
      const typename E::T a = E::from_f(v + 1.0f);      // + 1.0
      const typename E::T m = E::from_f(E::to_f(a) * 127.5f);  // * 127.5
      out[i * 3 + c] = static_cast<uint8_t>(static_cast<int>(E::to_f(m)));   // .to(uint8): truncation
    }
  }
}

// Antialiased bilinear resize of uint8 frames [T,H,W,3] -> [T,OH,OW,3] (torchvision `transforms.Resize(size)` on a uint8
// tensor, cvvae_inference_video.py:15-17,28: triangle filter whose support grows with the down-scale factor, window
// [int(c - s + 0.5), int(c + s + 0.5)) around c = scale * (i + 0.5), weights normalised to 1, result rounded half-up).
// fp32 weights and accumulation; torchvision's CPU path uses 16-bit fixed-point weights, so it differs from exact arithmetic -
// and from this kernel - by 1 LSB on < 1 % of the pixels (tests/test_gpu_ops.py).  One thread per output pixel (3 channels).
// out_f != nullptr: also apply `.half() / 127.5 - 1.0` and write [1,3,T,OH,OW] (the fused pre-processing of the script).
template <int DT>
__global__ void __launch_bounds__(256) resize_u8_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out_u8,
                                                        typename Elem<DT>::T* __restrict__ out_f, int T, int H, int W, int OH,
                                                        int OW, float sh, float sw) {
  using E = Elem<DT>;
  const long long n = 1ll * T * OH * OW;
  const float sup_h = sh >= 1.f ? sh : 1.f, inv_h = sh >= 1.f ? 1.f / sh : 1.f;
  const float sup_w = sw >= 1.f ? sw : 1.f, inv_w = sw >= 1.f ? 1.f / sw : 1.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % OW);
    const int oy = static_cast<int>((i / OW) % OH);
    const int t = static_cast<int>(i / (1ll * OW * OH));
    const float cy = sh * (oy + 0.5f), cx = sw * (ox + 0.5f);
    const int ymin = max(0, static_cast<int>(cy - sup_h + 0.5f));
    const int ysize = min(H, static_cast<int>(cy + sup_h + 0.5f)) - ymin;
    const int xmin = max(0, static_cast<int>(cx - sup_w + 0.5f));
    const int xsize = min(W, static_cast<int>(cx + sup_w + 0.5f)) - xmin;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, wsum_y = 0.f, wsum_x = 0.f;
    for (int a = 0; a < xsize; ++a) wsum_x += fmaxf(0.f, 1.f - fabsf((a + xmin - cx + 0.5f) * inv_w));
    const uint8_t* base = in + (1ll * t * H) * W * 3;
    for (int b = 0; b < ysize; ++b) {
      const float wy = fmaxf(0.f, 1.f - fabsf((b + ymin - cy + 0.5f) * inv_h));
      wsum_y += wy;
      const uint8_t* rowp = base + (1ll * (ymin + b) * W + xmin) * 3;
      float r0 = 0.f, r1 = 0.f, r2 = 0.f;
      for (int a = 0; a < xsize; ++a) {
        const float wx = fmaxf(0.f, 1.f - fabsf((a + xmin - cx + 0.5f) * inv_w));
        r0 = fmaf(wx, static_cast<float>(rowp[a * 3 + 0]), r0);
        r1 = fmaf(wx, static_cast<float>(rowp[a * 3 + 1]), r1);
        r2 = fmaf(wx, static_cast<float>(rowp[a * 3 + 2]), r2);
      }
      acc0 = fmaf(wy, r0, acc0);
      acc1 = fmaf(wy, r1, acc1);
      acc2 = fmaf(wy, r2, acc2);
    }
    const float norm = 1.f / (wsum_y * wsum_x);
    const float v[3] = {acc0 * norm, acc1 * norm, acc2 * norm};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float r = fminf(fmaxf(floorf(v[c] + 0.5f), 0.f), 255.f);
      if (out_u8) out_u8[i * 3 + c] = static_cast<uint8_t>(r);
      if (out_f) {
        const typename E::T h = E::from_f(r);
        const typename E::T q = E::from_f(E::to_f(h) / 127.5f);
        out_f[1ll * c * n + i] = E::from_f(E::to_f(q) - 1.0f);
      }
    }
  }
}

// One axis of torchvision's antialiased bilinear resize of a *float* tensor, as ATen's CPU kernel evaluates it
// (UpSampleKernel.cpp, _compute_indices_min_size_weights_aa with a float scalar type): centre c = scale * (i + 0.5) rounded
// to float, support s = max(scale, 1), window [int(c - s + 0.5), int(c + s + 0.5)) clipped to the input and to at most
// 2 * ceil(s) + 1 taps, triangle weights 1 - |(j - c + 0.5) * invscale| normalised by their float sum.  The `+ 0.5` and the
// product with invscale are double there (a float plus a double literal), so they are double here too, and every rounding
// ATen makes in fp32 is made here: the windows are the CPU kernel's and the weights differ from its by rounding order only.
struct AaAxis {
  float center, invscale, total;
  int lo, n;
  __device__ __forceinline__ AaAxis(int i, int in_size, float scale) {
    const float support = scale >= 1.f ? scale : 1.f;
    invscale = scale >= 1.f ? 1.f / scale : 1.f;
    // the double product of ATen is exact, so one rounding either way; the _rn intrinsics keep the compiler from fusing
    // the centre's product into the subtractions below (an unrounded centre moves windows and weights)
    center = __fmul_rn(scale, static_cast<float>(i) + 0.5f);
    lo = max(0, static_cast<int>(static_cast<double>(__fsub_rn(center, support)) + 0.5));
    n = min(in_size, static_cast<int>(static_cast<double>(__fadd_rn(center, support)) + 0.5)) - lo;
    n = min(max(n, 0), static_cast<int>(ceilf(support)) * 2 + 1);
    total = 0.f;
    for (int j = 0; j < n; ++j) total += raw(j);
  }
  __device__ __forceinline__ float raw(int j) const {
    const float d = __fsub_rn(static_cast<float>(j + lo), center);
    return fmaxf(0.f, 1.f - fabsf(static_cast<float>(__dmul_rn(__dadd_rn(d, 0.5), invscale))));
  }
  __device__ __forceinline__ float weight(int j) const { return total != 0.f ? raw(j) / total : raw(j); }
};

// The reference's training pre-processing of uint8 frames [T,H,W,3] (lvdm/data/decoder.py:99-109, transform.py): to float,
// antialiased bilinear resize to RH x RW, crop of OH x OW at (top, left), then (v / 255 - 0.5) * 2, all fp32, rounded once
// to the output type.  Output pixel (t, oy, ox) is pixel (oy + top, ox + left) of the resized frame, so the crop costs
// nothing.  Width is reduced first, then height, as ATen's separable kernel does (an axis whose size does not change gets
// the weights {1, 0}, which leaves it exact, as ATen's skipping of that axis does).  One thread per output pixel.
template <int DT>
__global__ void __launch_bounds__(256) train_input_kernel(const uint8_t* __restrict__ in, typename Elem<DT>::T* __restrict__ out,
                                                          int T, int H, int W, int top, int left, int OH, int OW, float sh,
                                                          float sw) {
  using E = Elem<DT>;
  const long long n = 1ll * T * OH * OW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % OW);
    const int oy = static_cast<int>((i / OW) % OH);
    const int t = static_cast<int>(i / (1ll * OW * OH));
    const AaAxis ay(oy + top, H, sh), ax(ox + left, W, sw);
    const uint8_t* base = in + ((1ll * t * H + ay.lo) * W + ax.lo) * 3;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
    for (int b = 0; b < ay.n; ++b) {
      const uint8_t* rowp = base + 1ll * b * W * 3;
      float r0 = 0.f, r1 = 0.f, r2 = 0.f;
      for (int a = 0; a < ax.n; ++a) {
        const float wx = ax.weight(a);
        r0 = fmaf(wx, static_cast<float>(rowp[a * 3 + 0]), r0);
        r1 = fmaf(wx, static_cast<float>(rowp[a * 3 + 1]), r1);
        r2 = fmaf(wx, static_cast<float>(rowp[a * 3 + 2]), r2);
      }
      const float wy = ay.weight(b);
      acc0 = fmaf(wy, r0, acc0);
      acc1 = fmaf(wy, r1, acc1);
      acc2 = fmaf(wy, r2, acc2);
    }
    const float v[3] = {acc0, acc1, acc2};
#pragma unroll
    for (int c = 0; c < 3; ++c) out[1ll * c * n + i] = E::from_f((v[c] / 255.f - 0.5f) * 2.f);
  }
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_video_train_input(const uint8_t* thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t RH,
                                       int32_t RW, int32_t top, int32_t left, int32_t OH, int32_t OW, int32_t dtype,
                                       void* stream) {
  CVVAE_CHECK_ARG(thwc && out_cthw && T > 0 && H > 0 && W > 0 && RH > 0 && RW > 0 && OH > 0 && OW > 0,
                  "cvvae_video_train_input: bad argument (T=%d H=%d W=%d RH=%d RW=%d OH=%d OW=%d)", T, H, W, RH, RW, OH, OW);
  CVVAE_CHECK_ARG(top >= 0 && left >= 0 && 1ll * top + OH <= RH && 1ll * left + OW <= RW,
                  "cvvae_video_train_input: crop %dx%d at (%d, %d) does not lie inside the %dx%d resized frame", OH, OW, top,
                  left, RH, RW);
  const long long n = 1ll * T * OH * OW;
  const unsigned blocks = static_cast<unsigned>(n / 256 + 1 < 16ll * num_sms() ? n / 256 + 1 : 16ll * num_sms());
  const float sh = static_cast<float>(H) / static_cast<float>(RH), sw = static_cast<float>(W) / static_cast<float>(RW);
  CVVAE_DISPATCH_DTYPE(dtype, {
    train_input_kernel<DT><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        thwc, reinterpret_cast<typename Elem<DT>::T*>(out_cthw), T, H, W, top, left, OH, OW, sh, sw);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_video_resize_u8(const uint8_t* thwc, uint8_t* out_thwc, void* out_cthw, int32_t T, int32_t H, int32_t W,
                                     int32_t OH, int32_t OW, int32_t dtype, void* stream) {
  CVVAE_CHECK_ARG(thwc && (out_thwc || out_cthw) && T > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "cvvae_video_resize_u8: bad argument");
  const long long n = 1ll * T * OH * OW;
  const unsigned blocks = static_cast<unsigned>(n / 256 + 1 < 16ll * num_sms() ? n / 256 + 1 : 16ll * num_sms());
  const float sh = static_cast<float>(H) / static_cast<float>(OH), sw = static_cast<float>(W) / static_cast<float>(OW);
  CVVAE_DISPATCH_DTYPE16(dtype, "video_io", {
    resize_u8_kernel<DT><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        thwc, out_thwc, reinterpret_cast<typename Elem<DT>::T*>(out_cthw), T, H, W, OH, OW, sh, sw);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_video_u8_to_f16(const uint8_t* thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t dtype,
                                     void* stream) {
  CVVAE_CHECK_ARG(thwc && out_cthw && T > 0 && H > 0 && W > 0, "cvvae_video_u8_to_f16: bad argument");
  const long long thw = 1ll * T * H * W;
  const unsigned blocks = static_cast<unsigned>(thw / 256 + 1 < 16ll * num_sms() ? thw / 256 + 1 : 16ll * num_sms());
  CVVAE_DISPATCH_DTYPE16(dtype, "video_io", {
    u8_to_f16_kernel<DT><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        thwc, reinterpret_cast<typename Elem<DT>::T*>(out_cthw), thw);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_video_f16_to_u8(const void* in_cthw, uint8_t* thwc, int32_t T, int32_t H, int32_t W, int32_t dtype,
                                     void* stream) {
  CVVAE_CHECK_ARG(thwc && in_cthw && T > 0 && H > 0 && W > 0, "cvvae_video_f16_to_u8: bad argument");
  const long long thw = 1ll * T * H * W;
  const unsigned blocks = static_cast<unsigned>(thw / 256 + 1 < 16ll * num_sms() ? thw / 256 + 1 : 16ll * num_sms());
  CVVAE_DISPATCH_DTYPE16(dtype, "video_io", {
    f16_to_u8_kernel<DT><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const typename Elem<DT>::T*>(in_cthw), thwc, thw);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
