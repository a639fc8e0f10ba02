// Data-movement kernels either side of the convolutions: replicate border fill of pre-padded buffers, generic strided
// copy (with a vectorised row path for the wrapper's tile assembly), and the tile blend of the wrapper.  All HBM-bound,
// coalesced on the channel axis, 128-bit accesses where the layout allows.  The movers are templated on the storage word U
// (uint16_t for f16 / bf16, uint32_t for fp32): a 16-byte vector carries 8 or 4 elements.
#include <type_traits>

#include "common.cuh"

namespace cvvae {

struct V5 {
  void* ptr;
  int B, T, H, W, C;
  long long s_b, s_t, s_h, s_w, s_c;
};
static V5 mk(const cvvae_tensor5* t) { return V5{t->ptr, t->B, t->T, t->H, t->W, t->C, t->s_b, t->s_t, t->s_h, t->s_w, t->s_c}; }

static bool vec8_ok(const cvvae_tensor5* t) {
  return t->s_c == 1 && t->C % 8 == 0 && t->s_w % 8 == 0 && t->s_h % 8 == 0 && t->s_t % 8 == 0 && t->s_b % 8 == 0 &&
         reinterpret_cast<uintptr_t>(t->ptr) % 16 == 0;
}

// word type of a dtype's storage
template <int DT>
using Word = typename std::conditional<sizeof(typename Elem<DT>::T) == 4, uint32_t, uint16_t>::type;

// frame of a pre-padded buffer <- nearest interior position
template <typename U>
__global__ void __launch_bounds__(256) replicate_border_kernel(const V5 x) {
  const int vecs = x.C / static_cast<int>(16 / sizeof(U));
  const int per_frame = 2 * x.W + 2 * (x.H - 2);  // border positions of one (b,t) image
  const long long n = 1ll * x.B * x.T * per_frame * vecs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int vi = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int e = static_cast<int>(r % per_frame); r /= per_frame;
    const int t = static_cast<int>(r % x.T);
    const int b = static_cast<int>(r / x.T);
    int h, w;
    if (e < x.W) { h = 0; w = e; }
    else if (e < 2 * x.W) { h = x.H - 1; w = e - x.W; }
    else {
      const int k = e - 2 * x.W;
      h = 1 + (k >> 1);
      w = (k & 1) ? x.W - 1 : 0;
    }
    const int hs = min(max(h, 1), x.H - 2), ws = min(max(w, 1), x.W - 2);
    U* base = reinterpret_cast<U*>(x.ptr) + b * x.s_b + t * x.s_t;
    const uint4 v = *(reinterpret_cast<const uint4*>(base + hs * x.s_h + ws * x.s_w) + vi);
    *(reinterpret_cast<uint4*>(base + h * x.s_h + w * x.s_w) + vi) = v;
  }
}

// element-wise strided copy; ROUND: fp32 storage, values rounded to the nearest TF32 value (the channel-padding copy of a
// network input, whose only consumer is the tensor-core convolution)
template <typename U, bool ROUND>
__global__ void __launch_bounds__(256) copy5_kernel(const V5 x, const V5 y) {
  const long long n = 1ll * y.B * y.T * y.H * y.W * y.C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // iterate in the order of the destination's fastest axis to keep stores coalesced
    long long r = i;
    int c, w, h, t, b;
    if (y.s_c == 1) {
      c = static_cast<int>(r % y.C); r /= y.C;
      w = static_cast<int>(r % y.W); r /= y.W;
      h = static_cast<int>(r % y.H); r /= y.H;
      t = static_cast<int>(r % y.T); r /= y.T;
      b = static_cast<int>(r);
    } else {
      w = static_cast<int>(r % y.W); r /= y.W;
      h = static_cast<int>(r % y.H); r /= y.H;
      t = static_cast<int>(r % y.T); r /= y.T;
      c = static_cast<int>(r % y.C); r /= y.C;
      b = static_cast<int>(r);
    }
    U v = c < x.C ? reinterpret_cast<const U*>(x.ptr)[b * x.s_b + t * x.s_t + h * x.s_h + w * x.s_w + c * x.s_c]
                  : static_cast<U>(0);  // channel zero-fill when the destination is wider
    if constexpr (ROUND) v = __float_as_uint(tf32_rn(__uint_as_float(v)));
    reinterpret_cast<U*>(y.ptr)[b * y.s_b + t * y.s_t + h * y.s_h + w * y.s_w + c * y.s_c] = v;
  }
}

// Both views contiguous along W (two NCDHW tensors described as [B,T,H,W,C] with s_w == 1): the wrapper's tile assembly
// - a cropped tile result copied into its window of the pre-allocated clip (modeling_vae.py:181-191,267-277,207-210).
// Rows are W contiguous elements; 128-bit accesses when both rows are 16-byte aligned, else element-wise.
template <typename U>
__global__ void __launch_bounds__(256) copy_rows_kernel(const V5 x, const V5 y, int vec) {
  const int wv = vec ? y.W / static_cast<int>(16 / sizeof(U)) : y.W;   // work items per row
  const long long n = 1ll * y.B * y.C * y.T * y.H * wv;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long r = i;
    const int w = static_cast<int>(r % wv); r /= wv;
    const int h = static_cast<int>(r % y.H); r /= y.H;
    const int t = static_cast<int>(r % y.T); r /= y.T;
    const int c = static_cast<int>(r % y.C); r /= y.C;
    const int b = static_cast<int>(r);
    const U* src = reinterpret_cast<const U*>(x.ptr) + b * x.s_b + t * x.s_t + h * x.s_h + c * x.s_c;
    U* dst = reinterpret_cast<U*>(y.ptr) + b * y.s_b + t * y.s_t + h * y.s_h + c * y.s_c;
    if (vec) reinterpret_cast<uint4*>(dst)[w] = __ldg(reinterpret_cast<const uint4*>(src) + w);
    else dst[w] = src[w];
  }
}

// Spatial taps packed into channels: y[b,t,h,w,(kh*KW+kw)*Cx + c] = x[b,t,h+kh+off_h,w+kw+off_w,c] (zero or clamped outside
// the image), channels beyond KH*KW*Cx zero.  Turns the KT x KH x KW convolution of a network INPUT (3 / 4 channels, where a
// 64-channel K block per tap would be 95 % zeros) into a KT x 1 x 1 convolution over KH*KW*Cx (<= 64) channels.
// One thread per (position, 8-channel vector) of y, consecutive threads walking w (coalesced 2-byte loads per tap through
// x's strides - the caller's NCDHW tensor - and coalesced 16-byte stores: one in 16-bit storage, two in fp32, where the
// values are rounded to the nearest TF32 value for the tensor-core convolution that reads them).  A thread's vector index is loop-invariant
// (the grid stride is a multiple of y.C/8), so the (dh, dw, channel) source of each of its 8 channels is resolved once.
// (A shared-memory staged variant measured slower: 1.75 vs 1.38 ms per step; the loads hit L1/L2, the stores dominate.)
template <typename U>
__global__ void __launch_bounds__(256) pack_taps_hw_kernel(const V5 x, const V5 y, int KH, int KW, int off_h, int off_w,
                                                           int replicate) {
  const int vecs = y.C >> 3;
  const long long n = 1ll * y.B * y.T * y.H * y.W * vecs;
  const int used = KH * KW * x.C;
  const long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int v = static_cast<int>(i0 % vecs);     // invariant: gridDim.x * 256 % vecs == 0 (vecs divides 256)
  int dh[8], dw[8];
  long long dc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = v * 8 + j;
    const int tap = ch < used ? ch / x.C : 0;
    dh[j] = ch < used ? tap / KW + off_h : -(1 << 20);   // far outside: contributes zero (never clamped: see below)
    dw[j] = tap % KW + off_w;
    dc[j] = ch < used ? (ch - tap * x.C) * x.s_c : 0;
  }
  for (long long i = i0; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long r = i / vecs;
    const int w = static_cast<int>(r % y.W); r /= y.W;
    const int h = static_cast<int>(r % y.H); r /= y.H;
    const int t = static_cast<int>(r % y.T); r /= y.T;
    const int b = static_cast<int>(r);
    const U* xb = reinterpret_cast<const U*>(x.ptr) + b * x.s_b + t * x.s_t;
    U o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int hi = h + dh[j], wi = w + dw[j];
      const bool pad_ch = dh[j] < -(1 << 19);
      bool ok = !pad_ch;
      if (replicate && ok) {
        hi = min(max(hi, 0), x.H - 1);
        wi = min(max(wi, 0), x.W - 1);
      } else {
        ok = ok && hi >= 0 && hi < x.H && wi >= 0 && wi < x.W;
      }
      o[j] = ok ? __ldg(xb + hi * x.s_h + wi * x.s_w + dc[j]) : static_cast<U>(0);
    }
    U* yp = reinterpret_cast<U*>(y.ptr) + b * y.s_b + t * y.s_t + h * y.s_h + w * y.s_w + v * 8;
    if constexpr (sizeof(U) == 4) {
      uint32_t r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = __float_as_uint(tf32_rn(__uint_as_float(o[j])));
      reinterpret_cast<uint4*>(yp)[0] = make_uint4(r[0], r[1], r[2], r[3]);
      reinterpret_cast<uint4*>(yp)[1] = make_uint4(r[4], r[5], r[6], r[7]);
    } else {
      uint4 pk;
      pk.x = o[0] | (static_cast<uint32_t>(o[1]) << 16);
      pk.y = o[2] | (static_cast<uint32_t>(o[3]) << 16);
      pk.z = o[4] | (static_cast<uint32_t>(o[5]) << 16);
      pk.w = o[6] | (static_cast<uint32_t>(o[7]) << 16);
      *reinterpret_cast<uint4*>(yp) = pk;
    }
  }
}

// b[.., i ..] = (1 - i/ov) * a[.., La-ov+i ..] + (i/ov) * b[.., i ..], fp32 math, one rounding
template <int DT>
__global__ void __launch_bounds__(256) blend_kernel(const V5 a, const V5 b, int ov, int axis) {
  using E = Elem<DT>;
  using T = typename E::T;
  const int H = axis == 1 ? ov : b.H;
  const int W = axis == 0 ? ov : b.W;
  const long long n = 1ll * b.B * b.T * H * W * b.C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long r = i;
    int c, w, h, t, bb;
    if (b.s_c == 1) {
      c = static_cast<int>(r % b.C); r /= b.C;
      w = static_cast<int>(r % W); r /= W;
      h = static_cast<int>(r % H); r /= H;
      t = static_cast<int>(r % b.T); r /= b.T;
      bb = static_cast<int>(r);
    } else {
      w = static_cast<int>(r % W); r /= W;
      h = static_cast<int>(r % H); r /= H;
      t = static_cast<int>(r % b.T); r /= b.T;
      c = static_cast<int>(r % b.C); r /= b.C;
      bb = static_cast<int>(r);
    }
    const int k = axis == 0 ? w : h;
    const float wb = __fdiv_rn(static_cast<float>(k), static_cast<float>(ov));
    const int ha = axis == 1 ? a.H - ov + h : h;
    const int wa = axis == 0 ? a.W - ov + w : w;
    const float av = E::to_f(reinterpret_cast<const T*>(a.ptr)[bb * a.s_b + t * a.s_t + ha * a.s_h + wa * a.s_w + c * a.s_c]);
    T* bp = reinterpret_cast<T*>(b.ptr) + bb * b.s_b + t * b.s_t + h * b.s_h + w * b.s_w + c * b.s_c;
    const float bv = E::to_f(*bp);
    // same three fp32 roundings as the reference's `(1 - w) * a + w * b` (no FMA contraction), then one to 16 bit
    *bp = E::from_f(__fadd_rn(__fmul_rn(__fsub_rn(1.0f, wb), av), __fmul_rn(wb, bv)));
  }
}

static unsigned grid_for(long long n) {
  long long blocks = (n + 255) / 256;
  const long long cap = 16ll * num_sms();
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_replicate_border(const cvvae_tensor5* xpad, int32_t dtype, void* stream) {
  CVVAE_CHECK_ARG(tensor_ok(xpad) && xpad->H >= 3 && xpad->W >= 3, "cvvae_replicate_border: bad argument");
  CVVAE_CHECK_ARG(vec8_ok(xpad), "cvvae_replicate_border: needs a 16-byte aligned channels-last view");
  CVVAE_DISPATCH_DTYPE(dtype, {
    using U = Word<DT>;
    const long long n = 1ll * xpad->B * xpad->T * (2 * xpad->W + 2 * (xpad->H - 2)) * (xpad->C / (16 / sizeof(U)));
    replicate_border_kernel<U><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(xpad));
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_copy5(const cvvae_tensor5* x, const cvvae_tensor5* y, int32_t dtype, void* stream) {
  CVVAE_CHECK_ARG(tensor_ok(x) && tensor_ok(y), "cvvae_copy5: null argument");
  CVVAE_CHECK_ARG(y->B == x->B && y->T == x->T && y->H == x->H && y->W == x->W && y->C >= x->C, "cvvae_copy5: shape mismatch");
  const long long n = 1ll * y->B * y->T * y->H * y->W * y->C;
  if (x->s_w == 1 && y->s_w == 1 && x->C == y->C && y->W > 1) {
    auto al8 = [](const cvvae_tensor5* t) {
      return t->s_h % 8 == 0 && t->s_t % 8 == 0 && t->s_b % 8 == 0 && t->s_c % 8 == 0 && reinterpret_cast<uintptr_t>(t->ptr) % 16 == 0;
    };
    const int vec = (y->W % 8 == 0 && al8(x) && al8(y)) ? 1 : 0;
    CVVAE_DISPATCH_DTYPE(dtype, {
      using U = Word<DT>;
      const long long per = 16 / sizeof(U);
      copy_rows_kernel<U><<<grid_for(vec ? n / per : n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(x), mk(y), vec);
    });
    CVVAE_LAUNCH_CHECK();
    return CVVAE_OK;
  }
  // a channels-first -> channels-last copy is the gather of a network input (the caller's NCDHW tensor) into the
  // channel-padded buffer of the first convolution, its only reader: in fp32 storage it stores TF32-rounded values
  const bool gather = x->s_c != 1 && y->s_c == 1;
  CVVAE_DISPATCH_DTYPE(dtype, {
    using U = Word<DT>;
    if constexpr (DT == CVVAE_F32) {
      if (gather) copy5_kernel<U, true><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(x), mk(y));
      else copy5_kernel<U, false><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(x), mk(y));
    } else {
      copy5_kernel<U, false><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(x), mk(y));
    }
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_pack_taps_hw(const cvvae_tensor5* x, const cvvae_tensor5* y, int32_t KH, int32_t KW, int32_t off_h,
                                  int32_t off_w, int32_t pad_hw, int32_t dtype, void* stream) {
  CVVAE_CHECK_ARG(tensor_ok(x) && tensor_ok(y) && KH >= 1 && KH <= 3 && KW >= 1 && KW <= 3, "cvvae_pack_taps_hw: bad argument");
  CVVAE_CHECK_ARG(y->B == x->B && y->T == x->T && y->C >= KH * KW * x->C, "cvvae_pack_taps_hw: y.C %d < %d taps x %d channels",
                  y->C, KH * KW, x->C);
  CVVAE_CHECK_ARG(vec8_ok(y), "cvvae_pack_taps_hw: y must be a 16-byte aligned channels-last view with C %% 8 == 0");
  const int vecs = y->C / 8;
  CVVAE_CHECK_ARG(vecs <= 32 && 256 % vecs == 0, "cvvae_pack_taps_hw: y.C = %d unsupported (C/8 must divide 256)", y->C);
  const long long n = 1ll * y->B * y->T * y->H * y->W * vecs;
  CVVAE_DISPATCH_DTYPE(dtype, {
    pack_taps_hw_kernel<Word<DT>><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        mk(x), mk(y), KH, KW, off_h, off_w, pad_hw == CVVAE_PAD_REPLICATE ? 1 : 0);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_blend(const cvvae_tensor5* a, const cvvae_tensor5* b, int32_t overlap, int32_t axis, int32_t dtype,
                           void* stream) {
  CVVAE_CHECK_ARG(tensor_ok(a) && tensor_ok(b) && overlap > 0 && (axis == 0 || axis == 1), "cvvae_blend: bad argument");
  CVVAE_CHECK_ARG(a->B == b->B && a->T == b->T && a->C == b->C, "cvvae_blend: shape mismatch");
  if (axis == 0) CVVAE_CHECK_ARG(a->H == b->H && a->W >= overlap && b->W >= overlap, "cvvae_blend: width overlap %d does not fit", overlap);
  if (axis == 1) CVVAE_CHECK_ARG(a->W == b->W && a->H >= overlap && b->H >= overlap, "cvvae_blend: height overlap %d does not fit", overlap);
  const long long n = 1ll * b->B * b->T * (axis == 1 ? overlap : b->H) * (axis == 0 ? overlap : b->W) * b->C;
  CVVAE_DISPATCH_DTYPE(dtype, { blend_kernel<DT><<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(mk(a), mk(b), overlap, axis); });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
