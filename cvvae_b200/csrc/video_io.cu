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

}  // namespace cvvae

using namespace cvvae;

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
