// CUDA-core direct convolution: the few layers the tensor-core path cannot take (3/4-channel network
// inputs read straight from the caller's NCDHW tensor, replicate H/W padding without a pre-padded
// buffer) and the on-device cross-check of conv_tc in the test-suite.  Any strides, any channel count.
// HBM-bound by design for its real uses (conv_in: K = 81, writes a 128-channel activation).
#include "common.cuh"

namespace cvvae {

static constexpr int kCoB = 16;  // output channels per thread

struct ConvDirectParams {
  const void* x;
  const void* w;
  const float* bias;
  const void* residual;
  void* y;
  int B, T_in, H_in, W_in, Cin, Cout;
  int T_out, H_out, W_out;
  long long xs_b, xs_t, xs_h, xs_w, xs_c;
  long long ys_b, ys_t, ys_h, ys_w, ys_c;
  int KT, KH, KW, st, sh, sw, off_t, off_h, off_w, pad_t, pad_hw, up_time, flags;
  float alpha;
  long long w_ld;
  long long P;  // output positions
};

template <int DT>
__global__ void __launch_bounds__(128) conv_direct_kernel(const ConvDirectParams p) {
  using E = Elem<DT>;
  using T = typename E::T;
  const long long pos = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pos >= p.P) return;
  const int co0 = blockIdx.y * kCoB;
  long long r = pos;
  const int wo = static_cast<int>(r % p.W_out); r /= p.W_out;
  const int ho = static_cast<int>(r % p.H_out); r /= p.H_out;
  const int to = static_cast<int>(r % p.T_out); r /= p.T_out;
  const int b = static_cast<int>(r);
  const T* __restrict__ x = reinterpret_cast<const T*>(p.x);
  const T* __restrict__ w = reinterpret_cast<const T*>(p.w);

  float acc[kCoB];
#pragma unroll
  for (int j = 0; j < kCoB; ++j) acc[j] = 0.f;

  for (int kt = 0; kt < p.KT; ++kt) {
    int ti = to * p.st + kt + p.off_t;
    if (ti < 0 || ti >= p.T_in) {
      if (p.pad_t == CVVAE_PAD_ZERO) continue;
      ti = ti < 0 ? 0 : p.T_in - 1;
    }
    for (int kh = 0; kh < p.KH; ++kh) {
      int hi = ho * p.sh + kh + p.off_h;
      if (hi < 0 || hi >= p.H_in) {
        if (p.pad_hw == CVVAE_PAD_ZERO) continue;
        hi = hi < 0 ? 0 : p.H_in - 1;
      }
      for (int kw = 0; kw < p.KW; ++kw) {
        int wi = wo * p.sw + kw + p.off_w;
        if (wi < 0 || wi >= p.W_in) {
          if (p.pad_hw == CVVAE_PAD_ZERO) continue;
          wi = wi < 0 ? 0 : p.W_in - 1;
        }
        const T* xp = x + b * p.xs_b + ti * p.xs_t + hi * p.xs_h + wi * p.xs_w;
        const int tap = (kt * p.KH + kh) * p.KW + kw;
        const T* wp = w + (static_cast<long long>(tap) * p.Cout + co0) * p.w_ld;
        for (int ci = 0; ci < p.Cin; ++ci) {
          const float xv = E::to_f(xp[ci * p.xs_c]);
#pragma unroll
          for (int j = 0; j < kCoB; ++j) {
            if (co0 + j < p.Cout) acc[j] = fmaf(xv, E::to_f(wp[static_cast<long long>(j) * p.w_ld + ci]), acc[j]);
          }
        }
      }
    }
  }

  const int chalf = p.up_time == 2 ? p.Cout / 2 : p.Cout;
  const long long m_index = pos;
#pragma unroll
  for (int j = 0; j < kCoB; ++j) {
    const int cg = co0 + j;
    if (cg >= p.Cout) break;
    int cc = cg, tt = to;
    if (p.up_time == 2) {
      const int n2 = cg / chalf;
      cc = cg - n2 * chalf;
      tt = 2 * to + n2 - 1;
      if (tt < 0) continue;
    }
    const long long o = b * p.ys_b + tt * p.ys_t + ho * p.ys_h + wo * p.ys_w + cc * p.ys_c;
    float a = acc[j] * p.alpha;
    if (p.bias) a += (p.flags & CVVAE_CONV_BIAS_ALONG_M) ? __ldg(p.bias + m_index) : __ldg(p.bias + cg);
    if (p.flags & CVVAE_CONV_OUT_F32) {
      reinterpret_cast<float*>(p.y)[o] = a;
    } else {
      if (p.residual) a += E::to_f(reinterpret_cast<const T*>(p.residual)[o]);
      reinterpret_cast<T*>(p.y)[o] = E::from_f(a);
    }
  }
}

int conv_direct_launch(const cvvae_conv_desc* d, cudaStream_t stream) {
  const cvvae_tensor5& x = d->x;
  const cvvae_tensor5& y = d->y;
  ConvDirectParams p{};
  p.x = x.ptr; p.w = d->w; p.bias = d->bias; p.residual = d->residual; p.y = y.ptr;
  p.B = x.B; p.T_in = x.T; p.H_in = x.H; p.W_in = x.W; p.Cin = x.C; p.Cout = d->Cout;
  p.up_time = d->up_time == 2 ? 2 : 1;
  p.T_out = p.up_time == 2 ? (y.T + 1) / 2 : y.T;
  p.H_out = y.H; p.W_out = y.W;
  p.xs_b = x.s_b; p.xs_t = x.s_t; p.xs_h = x.s_h; p.xs_w = x.s_w; p.xs_c = x.s_c;
  p.ys_b = y.s_b; p.ys_t = y.s_t; p.ys_h = y.s_h; p.ys_w = y.s_w; p.ys_c = y.s_c;
  p.KT = d->KT; p.KH = d->KH; p.KW = d->KW; p.st = d->st; p.sh = d->sh; p.sw = d->sw;
  p.off_t = d->off_t; p.off_h = d->off_h; p.off_w = d->off_w;
  p.pad_t = d->pad_t; p.pad_hw = d->pad_hw; p.flags = d->flags; p.alpha = d->alpha;
  p.w_ld = d->w_ld ? d->w_ld : x.C;
  CVVAE_CHECK_ARG(y.B == x.B, "conv: batch mismatch");
  CVVAE_CHECK_ARG(y.C == (p.up_time == 2 ? d->Cout / 2 : d->Cout), "conv: y.C %d inconsistent with Cout %d / up_time %d",
                  y.C, d->Cout, p.up_time);
  if ((d->flags & (CVVAE_CONV_W_PER_BATCH | CVVAE_CONV_X_SHARED)) || d->w2) {
    set_error("conv_direct: the batched-GEMM flags and the fused shortcut are tensor-core path features");
    return CVVAE_E_UNSUPPORTED;
  }
  if (d->gn_stats) {
    set_error("conv_direct: fused GroupNorm statistics are a tensor-core epilogue feature");
    return CVVAE_E_UNSUPPORTED;
  }
  p.P = 1ll * p.B * p.T_out * p.H_out * p.W_out;
  const long long gx = (p.P + 127) / 128;
  CVVAE_CHECK_ARG(gx > 0 && gx < (1ll << 31), "conv_direct: grid out of range");
  dim3 grid(static_cast<unsigned>(gx), static_cast<unsigned>((p.Cout + kCoB - 1) / kCoB));
  CVVAE_DISPATCH_DTYPE(d->dtype, { conv_direct_kernel<DT><<<grid, 128, 0, stream>>>(p); });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

// [Cout][Cin][taps] -> [taps][Cout][Cin]; fp32 weights are stored rounded to the nearest TF32 value, the precision the
// tensor cores multiply them in
template <int DT>
__global__ void pack_weight_kernel(const typename Elem<DT>::T* __restrict__ src, typename Elem<DT>::T* __restrict__ dst,
                                   int Cout, int Cin, int taps) {
  const long long n = 1ll * Cout * Cin * taps;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % Cin);
    const long long r = i / Cin;
    const int co = static_cast<int>(r % Cout);
    const int tap = static_cast<int>(r / Cout);
    const typename Elem<DT>::T v = src[(static_cast<long long>(co) * Cin + ci) * taps + tap];
    if constexpr (DT == CVVAE_F32) dst[i] = tf32_rn(v);
    else dst[i] = v;
  }
}

bool conv_tc_eligible(const cvvae_conv_desc* d, const char** why);
int conv_tc_launch(const cvvae_conv_desc* d, cudaStream_t stream);
int gn_stats_run(const cvvae_tensor5* x, int32_t groups, int32_t per_frame, int64_t* stats, int32_t dtype,
                 cudaStream_t stream, bool zero_first);

}  // namespace cvvae

extern "C" int cvvae_conv3d_direct(const cvvae_conv_desc* d, void* stream) {
  CVVAE_CHECK_ARG(d && cvvae::tensor_ok(&d->x) && cvvae::tensor_ok(&d->y) && d->w, "cvvae_conv3d_direct: null argument");
  return cvvae::conv_direct_launch(d, static_cast<cudaStream_t>(stream));
}

extern "C" int cvvae_conv3d(const cvvae_conv_desc* d, void* stream_) {
  CVVAE_CHECK_ARG(d && cvvae::tensor_ok(&d->x) && cvvae::tensor_ok(&d->y) && d->w, "cvvae_conv3d: null argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool tc = !(d->flags & CVVAE_CONV_FORCE_DIRECT) && cvvae::conv_tc_eligible(d, nullptr);
  if (!d->gn_stats) return tc ? cvvae::conv_tc_launch(d, stream) : cvvae::conv_direct_launch(d, stream);
  // consumer GroupNorm sums requested: fused in the tensor-core epilogue when that path can, otherwise one extra
  // statistics pass over y - either way `gn_stats` has y's sums added when the call returns
  if (tc) {
    const int rc = cvvae::conv_tc_launch(d, stream);
    if (rc != CVVAE_E_UNSUPPORTED) return rc;
  }
  cvvae_conv_desc plain = *d;
  plain.gn_stats = nullptr;
  int rc = tc ? cvvae::conv_tc_launch(&plain, stream) : cvvae::conv_direct_launch(&plain, stream);
  if (rc) return rc;
  return cvvae::gn_stats_run(&d->y, d->gn_groups, 0, d->gn_stats, d->dtype, stream, false);
}

extern "C" int cvvae_conv3d_is_tc(const cvvae_conv_desc* d) {
  if (!d || !cvvae::tensor_ok(&d->x) || !cvvae::tensor_ok(&d->y) || !d->w) return 0;
  return (!(d->flags & CVVAE_CONV_FORCE_DIRECT) && cvvae::conv_tc_eligible(d, nullptr)) ? 1 : 0;
}

extern "C" int cvvae_pack_conv_weight(const void* w_oikkk, void* w_packed, int32_t Cout, int32_t Cin, int32_t taps,
                                      int32_t dtype, void* stream) {
  CVVAE_CHECK_ARG(w_oikkk && w_packed && Cout > 0 && Cin > 0 && taps > 0, "cvvae_pack_conv_weight: bad argument");
  const long long n = 1ll * Cout * Cin * taps;
  const int blocks = static_cast<int>(n / 256 + 1 < 4096 ? n / 256 + 1 : 4096);
  CVVAE_DISPATCH_DTYPE(dtype, {
    using T = typename cvvae::Elem<DT>::T;
    cvvae::pack_weight_kernel<DT><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const T*>(w_oikkk), reinterpret_cast<T*>(w_packed), Cout, Cin, taps);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
