// Tap-stacked 3x3(x3) convolution for tiny Cout (the decoder's conv_out, 128 -> 3 at full resolution).
//
// With N = Cout padded to a minimal tile the tensor core is idle: every MMA still has to read its A tile from shared memory
// for a few cycles of math, and the ordinary kernel issues one such MMA per tap.
// Here the nine (kh,kw) taps are stacked along N instead: B = [9 taps x 8 channel slots (+8 pad) = 80 rows][64 K], and ONE
// MMA on the UNSHIFTED slab tile produces, for every slab position, the partial sums of all nine taps; only the time
// taps and the channel blocks remain in the K loop (KT x Cin/64 x 4 MMAs per sub-tile instead of 27 x ...).  The spatial
// shifts are applied afterwards, on the tiny per-position partials, through a shared-memory exchange:
//     y[h][w][c] = sum_{kh,kw} P[(kh,kw)][h+kh-1][w+kw-1][c].
// Tile: a 12 x 32 slab of input positions (384 MMA rows: 3 x 64 per MMA warpgroup) -> 10 x 30 outputs.
//
// Replaces cuDNN behind Decoder.conv_out (reference models/vae_models.py:942-944,999; vae_models3d_sd3.py:319,385).
#include "common.cuh"
#include "ptx.cuh"

namespace cvvae {

struct ConvStkParams {
  int B, T_in, T_out, H_out, W_out, Cin, Cout;
  int KT, off_t, off_h, off_w, pad_t;
  float alpha;
  int tiles_w, tiles_h, cblocks;
  const float* bias;
  void* y;
  long long ys_b, ys_t, ys_h, ys_w, ys_c;
  int xstride;  // floats per slab position in the exchange buffer
};

static constexpr int kSlabW = 32, kSlabH = 12, kOutW = 30, kOutH = 10;
static constexpr int kChunks = kSlabW * kSlabH / 128;   // 64-row MMA chunks per warpgroup (3 x 40 accumulator registers)
static constexpr int kNstk = 80;                      // 9 taps x 8 channel slots + 8 rows of padding
static constexpr uint32_t kSlabBytes = kSlabW * kSlabH * 128;  // 48 KB per 64-channel block
static constexpr uint32_t kBBytes = kNstk * 128;      // 10 KB
static constexpr int kNA = 2, kNB = 4;
static constexpr int kStkThreads = 384;               // warpgroup 0: TMA producers; 1, 2: MMA + epilogue

template <int DT>
__global__ void __launch_bounds__(kStkThreads, 1)
    conv_stk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvStkParams p) {
  using E = Elem<DT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + kNA * kSlabBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + kNB * kBBytes);
  uint64_t* fullA = bars;
  uint64_t* emptyA = bars + 4;
  uint64_t* fullB = bars + 8;
  uint64_t* emptyB = bars + 12;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int id = blockIdx.x;
  const int t = id % p.T_out; id /= p.T_out;
  const int w0 = (id % p.tiles_w) * kOutW; id /= p.tiles_w;
  const int h0 = (id % p.tiles_h) * kOutH;
  const int b = id / p.tiles_h;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kNA; ++i) { ptx::mbar_init(&fullA[i], 1); ptx::mbar_init(&emptyA[i], 2); }
    for (int i = 0; i < kNB; ++i) { ptx::mbar_init(&fullB[i], 1); ptx::mbar_init(&emptyB[i], 2); }
    ptx::fence_mbar_init();
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
  }
  __syncthreads();

  // the K loop: time taps (clamped or skipped at the clip ends) x 64-channel blocks
  auto for_each_step = [&](auto&& f) {
    for (int kt = 0; kt < p.KT; ++kt) {
      int ti = t + kt + p.off_t;
      if (ti < 0 || ti >= p.T_in) {
        if (p.pad_t == CVVAE_PAD_ZERO) continue;
        ti = ti < 0 ? 0 : p.T_in - 1;
      }
      for (int cb = 0; cb < p.cblocks; ++cb) f(kt, ti, cb);
    }
  };

  if (threadIdx.x < 128) {
    ptx::setmaxnreg_dec<40>();
    ptx::Ring r;
    if (warp == 0) {
      for_each_step([&](int kt, int ti, int cb) {
        ptx::mbar_wait(&emptyA[r.slot], r.phase ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&fullA[r.slot], kSlabBytes);
          // slab position (0,0) is the input position of output (h0,w0) at tap (0,0)
          ptx::tma_load_5d(sA + r.slot * kSlabBytes, &tmA, &fullA[r.slot], cb * 64, w0 + p.off_w, h0 + p.off_h, ti, b);
        }
        __syncwarp();
        r.advance(kNA);
      });
    } else if (warp == 1) {
      for_each_step([&](int kt, int ti, int cb) {
        ptx::mbar_wait(&emptyB[r.slot], r.phase ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&fullB[r.slot], kBBytes);
          ptx::tma_load_3d(sB + r.slot * kBBytes, &tmB, &fullB[r.slot], cb * 64, 0, kt);
        }
        __syncwarp();
        r.advance(kNB);
      });
    }
    return;
  }

  // ------------------------------------------------------------- MMA warpgroups: 192 slab positions (3 x 64 rows) each
  ptx::setmaxnreg_inc<232>();
  const int half = (threadIdx.x >> 7) - 1;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float acc[kChunks][kNstk / 2];
  {
    ptx::Ring ra, rb;
    int pendA = -1, pendB = -1;
    uint32_t accumulate = 0;
    for_each_step([&](int kt, int ti, int cb) {
      ptx::mbar_wait(&fullA[ra.slot], ra.phase);
      ptx::mbar_wait(&fullB[rb.slot], rb.phase);
      const int ch_left = p.Cin - cb * 64;
      const int ksteps = ch_left >= 64 ? 4 : (ch_left + 15) >> 4;
      const uint32_t a0 = ptx::smem_u32(sA + ra.slot * kSlabBytes) + static_cast<uint32_t>(half * kChunks * 64) * 128u;
      const uint32_t b0 = ptx::smem_u32(sB + rb.slot * kBBytes);
      ptx::wgmma_fence();
#pragma unroll
      for (int c = 0; c < kChunks; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < ksteps)
            ptx::Wgmma<DT, kNstk>::run(acc[c], ptx::wgmma_desc_sw128(a0 + c * 8192u + 32u * k), ptx::wgmma_desc_sw128(b0 + 32u * k),
                                       accumulate | static_cast<uint32_t>(k));
      accumulate = 1;
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();
      if (wg_leader && pendA >= 0) {
        ptx::mbar_arrive(&emptyB[pendB]);
        ptx::mbar_arrive(&emptyA[pendA]);
      }
      pendA = ra.slot;
      pendB = rb.slot;
      ra.advance(kNA);
      rb.advance(kNB);
    });
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < kChunks; ++c) ptx::fence_regs(acc[c]);
  }

  // ------------------------------------------------------------- epilogue, both MMA warpgroups
  ptx::named_bar_sync(1, 256);   // both warpgroups are done reading the A ring
  float* exch = reinterpret_cast<float*>(sA);  // [384 slab positions][xstride]
  {
    // phase 1: every slab position writes its 9 x Cout partial sums (column 8 * tap + channel slot of the accumulator)
    const int wl = warp & 3;
#pragma unroll
    for (int c = 0; c < kChunks; ++c)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int pos = (half * kChunks + c) * 64 + wl * 16 + (lane >> 2) + rr * 8;
        float* dst = exch + static_cast<size_t>(pos) * p.xstride;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ch = 2 * (lane & 3) + e;
            if (ch < p.Cout) dst[tap * p.Cout + ch] = acc[c][4 * tap + 2 * rr + e];
          }
      }
  }
  ptx::named_bar_sync(1, 256);
  {
    // phase 2: outputs gather the nine shifted partials.  384 slab positions over 256 threads.
    using T = typename E::T;
    T* yb = reinterpret_cast<T*>(p.y) + b * p.ys_b + t * p.ys_t;
    for (int pos = threadIdx.x - 128; pos < kSlabW * kSlabH; pos += 256) {
      const int r = pos / kSlabW, c = pos % kSlabW;
      if (r >= kOutH || c >= kOutW) continue;   // output (r,c) of the tile reads slab positions (r+kh, c+kw)
      const int ho = h0 + r, wo = w0 + c;
      if (ho >= p.H_out || wo >= p.W_out) continue;
      float acc4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const float* src = exch + static_cast<size_t>((r + kh) * kSlabW + (c + kw)) * p.xstride + (kh * 3 + kw) * p.Cout;
          for (int ch = 0; ch < p.Cout; ++ch) acc4[ch] += src[ch];
        }
      for (int ch = 0; ch < p.Cout; ++ch) {
        float a = acc4[ch] * p.alpha;
        if (p.bias) a += __ldg(p.bias + ch);
        yb[ho * p.ys_h + wo * p.ys_w + ch * p.ys_c] = E::from_f(a);
      }
    }
  }
}

}  // namespace cvvae

using namespace cvvae;

// w_stacked: [KT][80][Cin] (row = (kh*3+kw)*8 + c, rows with c >= Cout and rows 72..79 zero), activation dtype.
extern "C" int cvvae_conv3d_stacked(const cvvae_conv_desc* d, void* stream_) {
  CVVAE_CHECK_ARG(d && tensor_ok(&d->x) && tensor_ok(&d->y) && d->w, "cvvae_conv3d_stacked: null argument");
  const cvvae_tensor5& x = d->x;
  const cvvae_tensor5& y = d->y;
  CVVAE_CHECK_ARG(d->KH == 3 && d->KW == 3 && d->st == 1 && d->sh == 1 && d->sw == 1 && d->up_time != 2,
                  "cvvae_conv3d_stacked: needs a stride-1 (KT x) 3 x 3 convolution");
  CVVAE_CHECK_ARG(d->Cout >= 1 && d->Cout <= 4 && y.C == d->Cout, "cvvae_conv3d_stacked: Cout %d not in 1..4", d->Cout);
  CVVAE_CHECK_ARG(!d->residual && !d->gn_stats && !(d->flags & (CVVAE_CONV_OUT_F32 | CVVAE_CONV_BIAS_ALONG_M | CVVAE_CONV_RELU |
                                                                    CVVAE_CONV_TF32_OUT)),
                  "cvvae_conv3d_stacked: residual / statistics / fp32 output / ReLU are not supported");
  CVVAE_CHECK_ARG(tma_view(x, 2) && reinterpret_cast<uintptr_t>(d->w) % 16 == 0 && x.C % 8 == 0,
                  "cvvae_conv3d_stacked: input must be a 16-byte aligned channels-last view");
  if (d->pad_hw != CVVAE_PAD_ZERO) {
    const int hi_h = (y.H - 1) + 2 + d->off_h, hi_w = (y.W - 1) + 2 + d->off_w;
    CVVAE_CHECK_ARG(d->off_h >= 0 && d->off_w >= 0 && hi_h < x.H && hi_w < x.W,
                    "cvvae_conv3d_stacked: replicate H/W padding needs a pre-padded (framed) input");
  }
  ConvStkParams p{};
  p.B = x.B; p.T_in = x.T; p.T_out = y.T; p.H_out = y.H; p.W_out = y.W; p.Cin = x.C; p.Cout = d->Cout;
  p.KT = d->KT; p.off_t = d->off_t; p.off_h = d->off_h; p.off_w = d->off_w; p.pad_t = d->pad_t;
  p.alpha = d->alpha; p.bias = d->bias; p.y = y.ptr;
  p.ys_b = y.s_b; p.ys_t = y.s_t; p.ys_h = y.s_h; p.ys_w = y.s_w; p.ys_c = y.s_c;
  p.tiles_w = (p.W_out + kOutW - 1) / kOutW;
  p.tiles_h = (p.H_out + kOutH - 1) / kOutH;
  p.cblocks = (p.Cin + 63) / 64;
  p.xstride = (9 * p.Cout) | 1;  // odd stride: conflict-free for consecutive positions
  CUtensorMap tmA, tmB;
  const cuuint32_t box[5] = {64, kSlabW, kSlabH, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
  if (!act_map(&tmA, x, 2, box, estr) || !weight_map(&tmB, d->w, p.Cin, kNstk, p.KT, p.Cin, 2, 64, kNstk)) return CVVAE_E_ARG;
  const long long grid = 1ll * p.T_out * p.tiles_w * p.tiles_h * p.B;
  CVVAE_CHECK_ARG(grid > 0 && grid < (1ll << 31), "cvvae_conv3d_stacked: grid out of range");
  const size_t smem = 1024 + kNA * kSlabBytes + kNB * kBBytes + 256;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CVVAE_DISPATCH_DTYPE16(d->dtype, "cvvae_conv3d_stacked", {
    static PerDeviceOnce attr;
    if (attr.need()) {
      CVVAE_CUDA(cudaFuncSetAttribute(conv_stk_kernel<DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr.mark();
    }
    conv_stk_kernel<DT><<<static_cast<unsigned>(grid), kStkThreads, smem, stream>>>(tmA, tmB, p);
  });
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
