// Attention pieces that are not GEMMs.  The GEMMs of the attention blocks (q/k/v/proj 1x1 convs, S = q k^T,
// O = P v) run on the tcgen05 convolution kernel as 1x1x1 "flat" problems (see engine.py); here:
//   * row softmax  fp32 logits -> probabilities in the activation dtype (models/vae_models.py:456,518,607); in fp32
//     storage they feed only the O = P v product and are stored rounded to the nearest TF32 value
//   * temporal attention over the latent frames of one chunk (models/vae_models.py:573-587)
#include "common.cuh"

namespace cvvae {

// One CTA per row.  The row is cached in shared memory (one HBM read of the fp32 logits, one write); 128-bit loads
// and 64-bit (16-bit storage) / 128-bit (fp32) stores when the row start and leading dimensions allow (the engine's buffers
// always do), scalar otherwise.
template <int DT>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, long long ld_s, void* p_,
                                                           long long ld_p, int cols, int vec) {
  using E = Elem<DT>;
  extern __shared__ __align__(16) float row[];
  __shared__ float red[32];
  const long long r = blockIdx.x;
  const float* sp = s + r * ld_s;
  typename E::T* pp = reinterpret_cast<typename E::T*>(p_) + r * ld_p;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cols4 = vec ? (cols >> 2) : 0;           // float4 groups handled by the vector path
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols4; c += blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(sp) + c);
    reinterpret_cast<float4*>(row)[c] = v;
    m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
  for (int c = cols4 * 4 + threadIdx.x; c < cols; c += blockDim.x) {
    const float v = sp[c];
    row[c] = v;
    m = fmaxf(m, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols4; c += blockDim.x) {
    float4 v = reinterpret_cast<float4*>(row)[c];
    v.x = __expf(v.x - m); v.y = __expf(v.y - m); v.z = __expf(v.z - m); v.w = __expf(v.w - m);
    reinterpret_cast<float4*>(row)[c] = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  for (int c = cols4 * 4 + threadIdx.x; c < cols; c += blockDim.x) {
    const float e = __expf(row[c] - m);
    row[c] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int c = threadIdx.x; c < cols4; c += blockDim.x) {
    const float4 v = reinterpret_cast<float4*>(row)[c];
    if constexpr (DT == CVVAE_F32) {
      reinterpret_cast<float4*>(pp)[c] =
          make_float4(E::mma_in(v.x * inv), E::mma_in(v.y * inv), E::mma_in(v.z * inv), E::mma_in(v.w * inv));
    } else {
      uint2 o;
      o.x = E::pack2(v.x * inv, v.y * inv);
      o.y = E::pack2(v.z * inv, v.w * inv);
      reinterpret_cast<uint2*>(pp)[c] = o;
    }
  }
  for (int c = cols4 * 4 + threadIdx.x; c < cols; c += blockDim.x) pp[c] = E::from_f(E::mma_in(row[c] * inv));
}

struct TAttnParams {
  const void *q, *k, *v;
  void* o;
  int B, T, H, W, C;
  long long qs[4], ks[4], vs[4], os[4];  // b, t, h, w strides
  float scale;
};

// MAXT bounds the per-thread score array: 32 covers every chunked configuration (<= 5 latent frames per chunk with the
// default 16-frame chunks); the 128 / 512 instantiations (scores in local memory) serve en_de_n_frames_a_time=None,
// where the decoder mid-block sees every latent frame of the clip at once.
template <int DT, int MAXT>
__global__ void __launch_bounds__(128) attn_temporal_kernel(const TAttnParams p) {
  constexpr int kMaxT = MAXT;
  using E = Elem<DT>;
  using T = typename E::T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long pos = static_cast<long long>(blockIdx.x) * 4 + warp;
  const long long npos = 1ll * p.B * p.H * p.W;
  if (pos >= npos) return;
  const int w = static_cast<int>(pos % p.W);
  const int h = static_cast<int>((pos / p.W) % p.H);
  const int b = static_cast<int>(pos / (1ll * p.W * p.H));
  const T* qb = reinterpret_cast<const T*>(p.q) + b * p.qs[0] + h * p.qs[2] + w * p.qs[3];
  const T* kb = reinterpret_cast<const T*>(p.k) + b * p.ks[0] + h * p.ks[2] + w * p.ks[3];
  const T* vb = reinterpret_cast<const T*>(p.v) + b * p.vs[0] + h * p.vs[2] + w * p.vs[3];
  T* ob = reinterpret_cast<T*>(p.o) + b * p.os[0] + h * p.os[2] + w * p.os[3];
  const int vecs = p.C >> 3;
  for (int i = 0; i < p.T; ++i) {
    float sc[kMaxT];
    float mx = -INFINITY;
    for (int j = 0; j < p.T; ++j) {
      float d = 0.f;
      for (int vi = lane; vi < vecs; vi += 32) {
        float fa[8], fc[8];
        unpack8<DT>(ld8<DT>(qb + i * p.qs[1] + vi * 8), fa);
        unpack8<DT>(ld8<DT>(kb + j * p.ks[1] + vi * 8), fc);
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(fa[e], fc[e], d);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      d *= p.scale;
      sc[j] = d;
      mx = fmaxf(mx, d);
    }
    float sum = 0.f;
    for (int j = 0; j < p.T; ++j) {
      sc[j] = __expf(sc[j] - mx);
      sum += sc[j];
    }
    const float inv = 1.f / sum;
    for (int vi = lane; vi < vecs; vi += 32) {
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      for (int j = 0; j < p.T; ++j) {
        float fc[8];
        unpack8<DT>(ld8<DT>(vb + j * p.vs[1] + vi * 8), fc);
        const float pj = sc[j] * inv;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(pj, fc[e], acc[e]);
      }
      st8<DT>(ob + i * p.os[1] + vi * 8, pack8<DT>(acc));
    }
  }
}

}  // namespace cvvae

using namespace cvvae;

extern "C" int cvvae_softmax_rows(const float* s, int64_t ld_s, void* p, int64_t ld_p, int64_t rows, int32_t cols,
                                  int32_t dtype, void* stream_) {
  CVVAE_CHECK_ARG(s && p && rows > 0 && cols > 0 && ld_s >= cols && ld_p >= cols, "cvvae_softmax_rows: bad argument");
  CVVAE_CHECK_ARG(rows < (1ll << 31), "cvvae_softmax_rows: too many rows");
  const size_t smem = sizeof(float) * cols;
  CVVAE_CHECK_ARG(smem <= 200 * 1024, "cvvae_softmax_rows: %d columns exceed the shared-memory row cache", cols);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_DISPATCH_DTYPE(dtype, {
    static PerDeviceOnce attr;
    if (smem > 48 * 1024 && attr.need()) {
      CVVAE_CUDA(cudaFuncSetAttribute(softmax_rows_kernel<DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      attr.mark();
    }
    const int vec = (ld_s % 4 == 0) && (ld_p % 4 == 0) && (reinterpret_cast<uintptr_t>(s) % 16 == 0) &&
                    (reinterpret_cast<uintptr_t>(p) % (4 * sizeof(typename Elem<DT>::T)) == 0);
    softmax_rows_kernel<DT><<<static_cast<unsigned>(rows), 256, smem, stream>>>(s, ld_s, p, ld_p, cols, vec);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

extern "C" int cvvae_attn_temporal(const cvvae_tensor5* q, const cvvae_tensor5* k, const cvvae_tensor5* v,
                                   const cvvae_tensor5* o, int32_t dtype, void* stream_) {
  CVVAE_CHECK_ARG(tensor_ok(q) && tensor_ok(k) && tensor_ok(v) && tensor_ok(o), "cvvae_attn_temporal: null argument");
  CVVAE_CHECK_ARG(q->T <= 512, "cvvae_attn_temporal: %d latent frames in one chunk > 512 unsupported (use temporal chunking)", q->T);
  CVVAE_CHECK_ARG(q->C % 8 == 0, "cvvae_attn_temporal: C %% 8 != 0");
  const cvvae_tensor5* ts[4] = {q, k, v, o};
  for (int i = 0; i < 4; ++i) {
    CVVAE_CHECK_ARG(ts[i]->s_c == 1 && ts[i]->B == q->B && ts[i]->T == q->T && ts[i]->H == q->H && ts[i]->W == q->W &&
                        ts[i]->C == q->C,
                    "cvvae_attn_temporal: shape mismatch");
    CVVAE_CHECK_ARG((ts[i]->s_w % 8 == 0) && (ts[i]->s_h % 8 == 0) && (ts[i]->s_t % 8 == 0) && (ts[i]->s_b % 8 == 0) &&
                        reinterpret_cast<uintptr_t>(ts[i]->ptr) % 16 == 0,
                    "cvvae_attn_temporal: operand not 16-byte aligned");
  }
  TAttnParams p{};
  p.q = q->ptr; p.k = k->ptr; p.v = v->ptr; p.o = o->ptr;
  p.B = q->B; p.T = q->T; p.H = q->H; p.W = q->W; p.C = q->C;
  auto cp = [](long long* d, const cvvae_tensor5* t) { d[0] = t->s_b; d[1] = t->s_t; d[2] = t->s_h; d[3] = t->s_w; };
  cp(p.qs, q); cp(p.ks, k); cp(p.vs, v); cp(p.os, o);
  p.scale = 1.0f / sqrtf(static_cast<float>(q->C));
  const long long npos = 1ll * p.B * p.H * p.W;
  const long long blocks = (npos + 3) / 4;
  CVVAE_CHECK_ARG(blocks < (1ll << 31), "cvvae_attn_temporal: too many positions");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_DISPATCH_DTYPE(dtype, {
    if (q->T <= 32) attn_temporal_kernel<DT, 32><<<static_cast<unsigned>(blocks), 128, 0, stream>>>(p);
    else if (q->T <= 128) attn_temporal_kernel<DT, 128><<<static_cast<unsigned>(blocks), 128, 0, stream>>>(p);
    else attn_temporal_kernel<DT, 512><<<static_cast<unsigned>(blocks), 128, 0, stream>>>(p);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
