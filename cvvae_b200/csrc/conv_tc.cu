// Implicit-GEMM convolution on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers), operands
// staged by TMA straight from the channels-last activation tensor: no im2col buffer ever exists.
//
// GEMM view: M = output positions, N = Cout, K = taps x Cin.  One CTA owns an output patch of TH x TW positions of one
// output frame (TH = NACC * 128/TW) and BN output channels.  Each of its two MMA warpgroups owns one 64-row half of
// every 128-position sub-tile and keeps NACC accumulators of 64 x BN fp32 (NACC * BN = 256: 128 registers per thread),
// so every weight tile staged in shared memory feeds 2 * NACC MMAs, and every activation slab feeds all KH row-taps:
//
//   A slab  (one per kt, kw, channel block): the (TH+KH-1) x TW input window, shifted by kw, loaded by ONE 5-D TMA
//           box into a SWIZZLE_128B buffer [row][w][128 B of channels: 64 in 16-bit storage, 32 in fp32].  Because the slab pitch is exactly TW positions (a multiple
//           of 8 -> 1024 B), the A operand of row-tap kh / sub-tile s / half h is the same buffer at byte offset
//           ((s*ROWS + kh) * TW + 64h) * 128: a 1024-B aligned wgmma descriptor, no copy.  Zero padding in H/W is TMA
//           out-of-bounds fill; time padding is a coordinate clamp (replicate) or a skipped tap (zeros).  Strided
//           (down-sampling) convs use TMA element strides.
//   B tile  (one per tap, channel block): [BN][128 B] slice of the packed weights [tap][Cout][Cin].
// A channel block is fed by 4 MMAs of 32 B each: K = 16 (f16 / bf16) or K = 8 (fp32 storage, TF32 products).
//
// Warpgroups (384 threads): 0 = producers (warp 0 slabs, warp 1 weights; registers handed to the MMA warpgroups),
// 1 and 2 = MMA issue + epilogue (registers -> bias/alpha/residual -> stores in the activation dtype, with the time-interleave scatter of
// Upsample3D folded into the store address, and the consumer GroupNorm's statistics).  16-bit channels-last outputs are
// staged in the freed A ring and written by TMA stores; their residual is prefetched by TMA after the last slab.
//
// Replaces cuDNN behind CausalConv3d / nn.Conv3d / Conv2dWithExtraDim / Downsample3D / Upsample3D
// (reference: models/vae_models.py:198-340, models/vae_blocks3d_sd3.py:16-364); see include/cvvae_b200.h.
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"

namespace cvvae {

struct ConvTcParams {
  int B, T_in, T_out, H_out, W_out, Cin, Cout;
  int KT, KH, KW, st, sh, sw, off_t, off_h, off_w, pad_t;
  int up_time, flags;
  float alpha;
  // tiling
  int TW, ROWS, NACC, TH, N_cta, KHs, n_hgroups, slab_rows;
  int tiles_w, tiles_h, n_tiles_n, cblocks, flat;
  int NA, NB;
  uint32_t slab_bytes, slab_stride, b_bytes;
  // epilogue
  const float* bias;
  const void* residual;
  void* y;
  long long ys_b, ys_t, ys_h, ys_w, ys_c;
  int yC, vec2;        // vec2: channel pairs may be stored (and residual pairs loaded) as one 32-bit / 64-bit word
  int64_t* gn_stats;   // fused GroupNorm statistics of y
  int gn_groups, gn_cpg;
  // fused 1x1 shortcut (ResnetBlock3D nin_shortcut / conv_shortcut as extra K steps of conv2): cblocks2 channel blocks
  // of a second input tensor (same positions as the output) times a [Cout][Cin2] matrix, accumulated after the taps
  int Cin2, cblocks2;
  // epilogue through shared memory and TMA stores (16-bit channels-last outputs), residual prefetched into the A ring
  int tma_epi;
  unsigned long long* trace;  // optional [trace_n][8] globaltimer stamps per CTA (diagnostics)
  int trace_n;
};

static constexpr int kThreads = 384;
static constexpr int kProducerRegs = 40, kMmaRegs = 232;   // 128 * 40 + 256 * 232 <= 64 K registers
static constexpr uint32_t kBarBytes = 2048;                // barriers + GroupNorm bins after the operand rings

__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t parity) { ptx::mbar_wait(bar, parity); }

struct TileCoord {
  int b, t, h0, w0, n0;
};

__device__ __forceinline__ TileCoord decode_tile(const ConvTcParams& p) {
  int id = static_cast<int>(blockIdx.x);
  TileCoord c;
  c.n0 = (id % p.n_tiles_n) * p.N_cta;
  id /= p.n_tiles_n;
  c.t = id % p.T_out;
  id /= p.T_out;
  c.w0 = (id % p.tiles_w) * (p.flat ? p.NACC * 128 : p.TW);
  id /= p.tiles_w;
  c.h0 = (id % p.tiles_h) * p.TH;
  c.b = id / p.tiles_h;
  return c;
}

// Enumerate the activation-slab steps of one tile in the order every role agrees on.
// f(kt, ti, hg, kw, cb)
template <class F>
__device__ __forceinline__ void for_each_slab(const ConvTcParams& p, int t, F&& f) {
  for (int kt = 0; kt < p.KT; ++kt) {
    int ti = t * p.st + kt + p.off_t;
    if (ti < 0 || ti >= p.T_in) {
      if (p.pad_t == CVVAE_PAD_ZERO) continue;
      ti = ti < 0 ? 0 : p.T_in - 1;
    }
    for (int hg = 0; hg < p.n_hgroups; ++hg)
      for (int kw = 0; kw < p.KW; ++kw)
        for (int cb = 0; cb < p.cblocks; ++cb) f(kt, ti, hg, kw, cb);
  }
}

// TMA epilogue: channel block c (cb channels) of the tile.  Its first channel and frame in y, or false when it has nothing
// to write (past Cout, or the first half of the up_time = 2 interleave at t = 0).  A block never straddles the interleave
// halves (the plan asks for Cout / 2 to be a multiple of cb).
__device__ __forceinline__ bool epi_block(const ConvTcParams& p, const TileCoord& tc, int c, int cb, int& c0, int& t_o) {
  const int g = tc.n0 + c * cb;
  if (g >= p.Cout) return false;
  const int n_il = p.up_time == 2 ? g / (p.Cout / 2) : 0;
  c0 = g - n_il * (p.Cout / 2);
  t_o = p.up_time == 2 ? 2 * tc.t + n_il - 1 : tc.t;
  return t_o >= 0;
}
// TMA epilogue: the 64 positions s * 128 + 64 * hf of the tile (half hf of sub-tile s) are one box of the y / residual
// maps, {cb, TW, ROWS / 2} or {cb, 64, 1}; its (w, h) corner.
__device__ __forceinline__ void epi_piece(const ConvTcParams& p, const TileCoord& tc, int s, int hf, int& w, int& h) {
  if (p.flat) {
    w = tc.w0 + s * 128 + 64 * hf;
    h = 0;
  } else if (p.ROWS == 1) {
    w = tc.w0 + 64 * hf;
    h = tc.h0 + s;
  } else {
    w = tc.w0;
    h = tc.h0 + s * p.ROWS + hf * (p.ROWS / 2);
  }
}

template <int DT, int BN>
__global__ void __launch_bounds__(kThreads, 1)
    conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                   const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmR,
                   const ConvTcParams p) {
  constexpr int kMaxAcc = 256 / BN;   // 128-position sub-tiles per CTA at most
  constexpr int kR = BN / 2;          // accumulator registers per thread per sub-tile
  using E = Elem<DT>;
  // channels per 128-byte operand row (one channel block: 64 in 16-bit storage, 32 in fp32) and K per MMA (a quarter)
  constexpr int kCB = 128 / static_cast<int>(sizeof(typename E::T));
  constexpr int kKmma = kCB / 4;
  constexpr int kKshift = kKmma == 16 ? 4 : 3;   // log2(kKmma)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + static_cast<size_t>(p.NA) * p.slab_stride;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + static_cast<size_t>(p.NB) * p.b_bytes);
  uint64_t* fullA = bars;         // [8]
  uint64_t* emptyA = bars + 8;    // [8]
  uint64_t* fullB = bars + 16;    // [8]
  uint64_t* emptyB = bars + 24;   // [8]
  unsigned long long* gn_bins = reinterpret_cast<unsigned long long*>(bars + 64);  // [64 groups][2] fixed-point partial sums

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool traced = p.trace != nullptr && static_cast<int>(blockIdx.x) < p.trace_n;
  unsigned long long* trc = traced ? p.trace + static_cast<size_t>(blockIdx.x) * 8 : nullptr;
  if (traced && threadIdx.x == 0) trc[0] = ptx::globaltimer_ns();
  const TileCoord tc = decode_tile(p);
  // sub-tiles that contain at least one valid output position
  int nacc_eff;
  if (p.flat) {
    nacc_eff = min(p.NACC, (p.W_out - tc.w0 + 127) / 128);
  } else {
    nacc_eff = max(0, min(p.NACC, (p.H_out - tc.h0 + p.ROWS - 1) / p.ROWS));
  }

  if (threadIdx.x < 128) gn_bins[threadIdx.x] = 0ull;
  if (threadIdx.x == 0) {
    for (int i = 0; i < p.NA; ++i) {
      ptx::mbar_init(&fullA[i], 1);
      ptx::mbar_init(&emptyA[i], 2);   // one arrival per MMA warpgroup
    }
    for (int i = 0; i < p.NB; ++i) {
      ptx::mbar_init(&fullB[i], 1);
      ptx::mbar_init(&emptyB[i], 2);
    }
    ptx::fence_mbar_init();
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (p.tma_epi) {
      ptx::prefetch_tmap(&tmY);
      if (p.residual) ptx::prefetch_tmap(&tmR);
    }
  }
  __syncthreads();
  if (traced && threadIdx.x == 0) trc[1] = ptx::globaltimer_ns();

  if (threadIdx.x < 128) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    // The whole warp walks the step sequence (every operand of the TMA instruction is warp-uniform); one elected lane
    // issues.  Warps 2 and 3 have nothing to do.
    int slot = 0;
    uint32_t phase = 0;
    auto advance = [&](int n) {
      __syncwarp();
      if (++slot == n) {
        slot = 0;
        phase ^= 1;
      }
    };
    if (warp == 0) {
      // ------------------------------------------------------------- A producer
      const int xb = (p.flags & CVVAE_CONV_X_SHARED) ? 0 : tc.b;  // batched GEMM with one shared left operand
      for_each_slab(p, tc.t, [&](int kt, int ti, int hg, int kw, int cb) {
        wait_bar(&emptyA[slot], phase ^ 1);
        uint8_t* dst = sA + static_cast<size_t>(slot) * p.slab_stride;
        if (ptx::elect_one()) {
          if (p.flat) {
            ptx::mbar_expect_tx(&fullA[slot], static_cast<uint32_t>(nacc_eff) * 128u * 128u);
            for (int s = 0; s < nacc_eff; ++s)
              ptx::tma_load_5d(dst + s * 16384, &tmA, &fullA[slot], cb * kCB, tc.w0 + s * 128, 0, ti, xb);
          } else {
            ptx::mbar_expect_tx(&fullA[slot], p.slab_bytes);
            ptx::tma_load_5d(dst, &tmA, &fullA[slot], cb * kCB, tc.w0 * p.sw + kw + p.off_w,
                             tc.h0 * p.sh + hg * p.KHs + p.off_h, ti, xb);
          }
        }
        advance(p.NA);
      });
      // fused 1x1 shortcut: the (unshifted) window of the second input, one slab per channel block
      for (int cb2 = 0; cb2 < p.cblocks2; ++cb2) {
        wait_bar(&emptyA[slot], phase ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&fullA[slot], p.slab_bytes);
          ptx::tma_load_5d(sA + static_cast<size_t>(slot) * p.slab_stride, &tmA2, &fullA[slot], cb2 * kCB, tc.w0, tc.h0, tc.t, xb);
        }
        advance(p.NA);
      }
      // TMA epilogue: claim the slots the epilogue stages the output in, one channel block per slot, and load the
      // block's residual into it.  A slot is released as soon as both MMA warpgroups have finished reading its slab,
      // which for all but the last slab happens while later slabs are multiplied: the residual arrives under the MMAs,
      // and a block's staging never waits for the other warpgroup's last MMAs unless it reuses the last slab's slot.
      if (kCB == 64 && p.tma_epi) {
        for (int c = 0; c < BN / kCB; ++c) {
          int c0, t_o;
          if (epi_block(p, tc, c, kCB, c0, t_o)) {
            wait_bar(&emptyA[slot], phase ^ 1);
            if (ptx::elect_one()) {
              uint8_t* dst = sA + static_cast<size_t>(slot) * p.slab_stride;
              if (p.residual) {
                ptx::mbar_expect_tx(&fullA[slot], static_cast<uint32_t>(nacc_eff) * 16384u);
                for (int s = 0; s < nacc_eff; ++s)
                  for (int hf = 0; hf < 2; ++hf) {
                    int w, h;
                    epi_piece(p, tc, s, hf, w, h);
                    ptx::tma_load_5d(dst + s * 16384 + hf * 8192, &tmR, &fullA[slot], c0, w, h, t_o, tc.b);
                  }
              } else {
                ptx::mbar_arrive(&fullA[slot]);
              }
            }
          }
          advance(p.NA);
        }
      }
    } else if (warp == 1) {
      // ------------------------------------------------------------- B producer
      for_each_slab(p, tc.t, [&](int kt, int ti, int hg, int kw, int cb) {
        for (int khs = 0; khs < p.KHs; ++khs) {
          // batched GEMM: the "tap" axis of the weight tensor indexes the batch item (1x1x1 problems only)
          const int tap = (p.flags & CVVAE_CONV_W_PER_BATCH) ? tc.b : (kt * p.KH + hg * p.KHs + khs) * p.KW + kw;
          wait_bar(&emptyB[slot], phase ^ 1);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(&fullB[slot], p.b_bytes);
            ptx::tma_load_3d(sB + static_cast<size_t>(slot) * p.b_bytes, &tmB, &fullB[slot], cb * kCB, tc.n0, tap);
          }
          advance(p.NB);
        }
      });
      for (int cb2 = 0; cb2 < p.cblocks2; ++cb2) {   // shortcut weights [Cout][Cin2]
        wait_bar(&emptyB[slot], phase ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&fullB[slot], p.b_bytes);
          ptx::tma_load_3d(sB + static_cast<size_t>(slot) * p.b_bytes, &tmB2, &fullB[slot], cb2 * kCB, tc.n0, 0);
        }
        advance(p.NB);
      }
    }
    return;
  }

  // ------------------------------------------------------------- MMA warpgroups
  ptx::setmaxnreg_inc<kMmaRegs>();
  const int half = (threadIdx.x >> 7) - 1;           // which 64-row half of every sub-tile
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float acc[kMaxAcc][kR];   // written first by an MMA with scale_d = 0; sub-tiles past nacc_eff are never read
  int epi_slot;             // the A-ring slot after the last slab, and its phase: where the TMA epilogue's blocks start
  uint32_t epi_phase;
  {
    int slotA = 0, slotB = 0;
    uint32_t phaseA = 0, phaseB = 0;
    int pendA = -1, pendB = -1;   // slots read by the MMA group still in flight, released once it completes
    bool first = true;
    uint32_t accumulate = 0;
    const uint32_t sub_stride = p.flat ? 16384u : static_cast<uint32_t>(p.ROWS * p.TW) * 128u;
    const uint32_t tap_stride = static_cast<uint32_t>(p.TW) * 128u;
    const uint32_t half_off = static_cast<uint32_t>(half) * 8192u;
    // one MMA group: every sub-tile x K step of the current weight tile against the slab rows starting at a_base
    auto mma_group = [&](uint32_t a_base, int ksteps, bool last_of_slab) {
      wait_bar(&fullB[slotB], phaseB);
      if (traced && first && threadIdx.x == 128) trc[3] = ptx::globaltimer_ns();
      first = false;
      const uint32_t b_base = ptx::smem_u32(sB + static_cast<size_t>(slotB) * p.b_bytes);
      if (nacc_eff == kMaxAcc && ksteps == 4) {
        // Full tile, nearly all of the work.  Fence, chain and commit sit in one basic block with no branch between the
        // MMAs, so ptxas issues the chain behind one warpgroup.arrive and closes the group on its last MMA.  Behind a
        // runtime branch every MMA gets its own arrive and group and the commit becomes a dummy MMA, so wait_group 1
        // below would wait for all of this group's real MMAs.
        ptx::wgmma_fence();
#pragma unroll
        for (int s = 0; s < kMaxAcc; ++s) {
          const uint32_t a_s = a_base + static_cast<uint32_t>(s) * sub_stride;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            ptx::Wgmma<DT, BN>::run(acc[s], ptx::wgmma_desc_sw128(a_s + 32u * k), ptx::wgmma_desc_sw128(b_base + 32u * k),
                                    accumulate | static_cast<uint32_t>(k));
        }
        ptx::wgmma_commit();
      } else {
        ptx::wgmma_fence();
#pragma unroll
        for (int s = 0; s < kMaxAcc; ++s) {
          if (s < nacc_eff) {
            const uint32_t a_s = a_base + static_cast<uint32_t>(s) * sub_stride;
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (k < ksteps)   // K = kKmma per MMA; channels beyond Cin are TMA zero-fill in both operands, skip those MMAs
                ptx::Wgmma<DT, BN>::run(acc[s], ptx::wgmma_desc_sw128(a_s + 32u * k), ptx::wgmma_desc_sw128(b_base + 32u * k),
                                        accumulate | static_cast<uint32_t>(k));
          }
        }
        ptx::wgmma_commit();
      }
      accumulate = 1;
      ptx::wgmma_wait<1>();   // the previous group is done reading its operands
      if (wg_leader) {
        if (pendB >= 0) ptx::mbar_arrive(&emptyB[pendB]);
        if (pendA >= 0) ptx::mbar_arrive(&emptyA[pendA]);
      }
      pendB = slotB;
      pendA = last_of_slab ? slotA : -1;
      if (++slotB == p.NB) {
        slotB = 0;
        phaseB ^= 1;
      }
    };
    auto next_slab = [&]() {
      if (++slotA == p.NA) {
        slotA = 0;
        phaseA ^= 1;
      }
    };
    for_each_slab(p, tc.t, [&](int kt, int ti, int hg, int kw, int cb) {
      wait_bar(&fullA[slotA], phaseA);
      if (traced && slotA == 0 && phaseA == 0 && threadIdx.x == 128) trc[2] = ptx::globaltimer_ns();
      const int ch_left = p.Cin - cb * kCB;
      const int ksteps = ch_left >= kCB ? 4 : (ch_left + kKmma - 1) >> kKshift;
      const uint32_t a0 = ptx::smem_u32(sA + static_cast<size_t>(slotA) * p.slab_stride) + half_off;
      for (int khs = 0; khs < p.KHs; ++khs) mma_group(a0 + static_cast<uint32_t>(khs) * tap_stride, ksteps, khs == p.KHs - 1);
      next_slab();
    });
    for (int cb2 = 0; cb2 < p.cblocks2; ++cb2) {   // fused 1x1 shortcut: row-tap 0 of the unshifted window
      wait_bar(&fullA[slotA], phaseA);
      const int ch_left = p.Cin2 - cb2 * kCB;
      const int ksteps = ch_left >= kCB ? 4 : (ch_left + kKmma - 1) >> kKshift;
      mma_group(ptx::smem_u32(sA + static_cast<size_t>(slotA) * p.slab_stride) + half_off, ksteps, true);
      next_slab();
    }
    if (traced && threadIdx.x == 128) trc[4] = ptx::globaltimer_ns();
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int s = 0; s < kMaxAcc; ++s) ptx::fence_regs(acc[s]);
    if (wg_leader) {
      if (pendB >= 0) ptx::mbar_arrive(&emptyB[pendB]);
      if (pendA >= 0) ptx::mbar_arrive(&emptyA[pendA]);
    }
    epi_slot = slotA;
    epi_phase = phaseA;
  }
  if (traced && threadIdx.x == 128) trc[5] = ptx::globaltimer_ns();

  // ------------------------------------------------------------- epilogue
  // Thread (warp wl of the warpgroup, lane) holds rows m = 64*half + 16*wl + lane/4 (+8) of every sub-tile and the
  // channel pairs n = 8j + 2*(lane%4) (+1).
  {
    using T = typename E::T;
    const int wl = warp & 3;
    const int cpair = 2 * (lane & 3);
    const int chalf = p.up_time == 2 ? p.Cout / 2 : p.Cout;
    const int bias_b = (p.flags & CVVAE_CONV_W_PER_BATCH) ? 0 : tc.b;  // batched GEMM: a row bias is shared by the batch items
    const bool bias_m = p.bias && (p.flags & CVVAE_CONV_BIAS_ALONG_M);
    const bool out_f32 = (p.flags & CVVAE_CONV_OUT_F32) != 0;
    // per row: offset of (b, h, w) in y, validity, bias along M
    long long roff[kMaxAcc][2];
    bool rok[kMaxAcc][2];
    float rbias[kMaxAcc][2];
#pragma unroll
    for (int s = 0; s < kMaxAcc; ++s) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = half * 64 + wl * 16 + (lane >> 2) + rr * 8;
        int h, w;
        if (p.flat) {
          h = 0;
          w = tc.w0 + s * 128 + m;
        } else {
          h = tc.h0 + s * p.ROWS + m / p.TW;
          w = tc.w0 + m % p.TW;
        }
        rok[s][rr] = s < nacc_eff && h < p.H_out && w < p.W_out;
        roff[s][rr] = tc.b * p.ys_b + h * p.ys_h + w * p.ys_w;
        rbias[s][rr] = 0.f;
        if (bias_m && rok[s][rr]) {
          const long long m_index =
              ((static_cast<long long>(bias_b) * p.T_out + tc.t) * p.H_out + h) * static_cast<long long>(p.W_out) + w;
          rbias[s][rr] = __ldg(p.bias + m_index);
        }
      }
    }
    // the consumer GroupNorm's statistics of channel pair (cc, cc + 1): reduce over the rows of the warp, add to the bins
    auto gn_add = [&](float gs0, float gq0, float gs1, float gq1, int cc, bool tok, bool c1ok) {
      // rows: lanes with the same lane%4 hold the same channels
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        gs0 += __shfl_xor_sync(0xffffffffu, gs0, o);
        gq0 += __shfl_xor_sync(0xffffffffu, gq0, o);
        gs1 += __shfl_xor_sync(0xffffffffu, gs1, o);
        gq1 += __shfl_xor_sync(0xffffffffu, gq1, o);
      }
      if (p.gn_cpg == 1) {
        if (lane < 4 && tok) {
          atomicAdd(&gn_bins[cc * 2], gn_fix(gs0, kGnSumScale));
          atomicAdd(&gn_bins[cc * 2 + 1], gn_fix(gq0, kGnSqScale));
          if (c1ok) {
            atomicAdd(&gn_bins[(cc + 1) * 2], gn_fix(gs1, kGnSumScale));
            atomicAdd(&gn_bins[(cc + 1) * 2 + 1], gn_fix(gq1, kGnSqScale));
          }
        }
      } else {
        float ts = gs0 + gs1, tq = gq0 + gq1;
        // channel pairs of one group are neighbouring lanes (lane%4)
        for (int o = 1; o < (p.gn_cpg >> 1) && o < 4; o <<= 1) {
          ts += __shfl_xor_sync(0xffffffffu, ts, o);
          tq += __shfl_xor_sync(0xffffffffu, tq, o);
        }
        const int lanes_per_group = min(p.gn_cpg >> 1, 4);
        // a group's channels never straddle the interleave halves (chalf is a multiple of the group size), so the
        // first lane of the group has the validity of all of them
        if (lane < 4 && (lane % lanes_per_group) == 0 && tok) {
          atomicAdd(&gn_bins[(cc / p.gn_cpg) * 2], gn_fix(ts, kGnSumScale));
          atomicAdd(&gn_bins[(cc / p.gn_cpg) * 2 + 1], gn_fix(tq, kGnSqScale));
        }
      }
    };
    // Interior tiles (every row and channel valid, output in the activation dtype stored as channel-pair words, bias along N) take a
    // loop without per-element tests.  The general loop's branches kept ptxas from batching the bias / residual loads
    // and the stores, so its epilogue took a third of a CTA's time.  Same operations in the same order: same bits.
    const bool tma_epi = kCB == 64 && p.tma_epi;
    const bool interior = nacc_eff == kMaxAcc && tc.n0 + BN <= p.Cout && !out_f32 && p.vec2 && !bias_m &&
                          (p.flat ? tc.w0 + kMaxAcc * 128 <= p.W_out
                                  : tc.h0 + kMaxAcc * p.ROWS <= p.H_out && tc.w0 + p.TW <= p.W_out);
    if (tma_epi) {
      if constexpr (kCB == 64) {
        // Every tile, interior or edge.  Channel block c of the tile (64 channels x NACC * 128 positions, 128-B rows in
        // SWIZZLE_128B order, i.e. the layout of the y map's boxes) is staged in A-ring slot epi_slot + c, which the A
        // producer hands over through fullA once both warpgroups have released it, with the block's residual loaded
        // when there is one; each thread reads its residual words and writes the result over them.  Then the
        // warpgroup's rows go out as TMA stores, which clip whatever lies outside y: edge rows, channels past Cout.
        // Same operations in the same order as the loops below: same bits.
        constexpr int kBlocks = BN / kCB;
        const int sw = lane >> 2;   // position & 7 of this thread's rows: the 16-byte chunk swizzle
        const uint32_t row_off = static_cast<uint32_t>(half * 64 + wl * 16 + sw) * 128u + 4u * (lane & 3);
        // The bias is loaded once, all loads in flight together: lane l holds channels n0 + 64c + 8(l/4) + 2(l%4) (+1),
        // and the thread's channel pair j = 8c + jj comes from lane 4jj + l%4.  A load per j, issued after the previous
        // j's work, left the loop waiting on L2 once per j.
        float bl[kBlocks][2];
#pragma unroll
        for (int c = 0; c < kBlocks; ++c) {
          const int ch = tc.n0 + c * kCB + 8 * sw + cpair;
          bl[c][0] = p.bias && ch < p.Cout ? __ldg(p.bias + ch) : 0.f;
          bl[c][1] = p.bias && ch + 1 < p.Cout ? __ldg(p.bias + ch + 1) : 0.f;
        }
        // Residual, statistics and a full set of sub-tiles are template switches of the staging loop, so that each
        // instance is straight-line code: with runtime tests inside, every pair carried predicate juggling and the
        // statistics arithmetic, and the loop issued several times the instructions it needs.
        auto stage_blocks = [&](auto res_c, auto gn_c, auto full_c) {
          constexpr bool kRes = decltype(res_c)::value, kGn = decltype(gn_c)::value, kFull = decltype(full_c)::value;
#pragma unroll
          for (int c = 0; c < kBlocks; ++c) {
            int c0, t_o;
            if (!epi_block(p, tc, c, kCB, c0, t_o)) continue;   // warp-uniform
            const int slot = epi_slot + c < p.NA ? epi_slot + c : epi_slot + c - p.NA;
            const uint32_t stage = ptx::smem_u32(sA + static_cast<size_t>(slot) * p.slab_stride) + row_off;
            wait_bar(&fullA[slot], epi_slot + c < p.NA ? epi_phase : epi_phase ^ 1);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * c + jj;
              const float b0 = __shfl_sync(0xffffffffu, bl[c][0], 4 * jj + (lane & 3));
              const float b1 = __shfl_sync(0xffffffffu, bl[c][1], 4 * jj + (lane & 3));
              const uint32_t chunk = stage + static_cast<uint32_t>((jj ^ sw) << 4);
              float gs0 = 0.f, gq0 = 0.f, gs1 = 0.f, gq1 = 0.f;
#pragma unroll
              for (int s = 0; s < kMaxAcc; ++s) {
                // sub-tiles past nacc_eff hold no output (and past NACC have no slot space)
                const bool sok = kFull || s < nacc_eff;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                  const uint32_t addr = chunk + static_cast<uint32_t>(s * 16384 + rr * 1024);
                  float a0 = fmaf(acc[s][4 * j + 2 * rr], p.alpha, b0);
                  float a1 = fmaf(acc[s][4 * j + 2 * rr + 1], p.alpha, b1);
                  if (kRes && sok) {
                    const float2 rf = E::to_f2(ptx::ld_shared_b32(addr));
                    a0 += rf.x;
                    a1 += rf.y;
                  }
                  const uint32_t o = E::pack2(a0, a1);
                  if (sok) ptx::st_shared_b32(addr, o);
                  if (kGn && rok[s][rr]) {
                    const float2 of = E::to_f2(o);
                    gs0 += of.x;
                    gq0 = fmaf(of.x, of.x, gq0);
                    gs1 += of.y;
                    gq1 = fmaf(of.y, of.y, gq1);
                  }
                }
              }
              // channels past Cout (a block that Cout ends inside; Cout % 8 == 0, so per pair) are computed from zero
              // weights and bias, clipped by the store and kept out of the statistics
              if (kGn) gn_add(gs0, gq0, gs1, gq1, c0 + 8 * jj + cpair, tc.n0 + 8 * j < p.Cout, true);
            }
          }
        };
        auto by_full = [&](auto res_c, auto gn_c) {
          if (nacc_eff == kMaxAcc) stage_blocks(res_c, gn_c, std::true_type{});
          else stage_blocks(res_c, gn_c, std::false_type{});
        };
        auto by_gn = [&](auto res_c) {
          if (p.gn_stats) by_full(res_c, std::true_type{});
          else by_full(res_c, std::false_type{});
        };
        if (p.residual) by_gn(std::true_type{});
        else by_gn(std::false_type{});
        ptx::fence_proxy_async();             // the staged words are visible to the TMA unit
        if (half == 0) ptx::named_bar_sync(3, 128);   // this warpgroup's rows are all written
        else ptx::named_bar_sync(4, 128);
        if (wg_leader) {
          for (int c = 0; c < kBlocks; ++c) {
            int bc0, bt;
            if (!epi_block(p, tc, c, kCB, bc0, bt)) continue;
            const int slot = epi_slot + c < p.NA ? epi_slot + c : epi_slot + c - p.NA;
            const uint8_t* src = sA + static_cast<size_t>(slot) * p.slab_stride + half * 8192;
            for (int s = 0; s < nacc_eff; ++s) {
              int w, h;
              epi_piece(p, tc, s, half, w, h);
              ptx::tma_store_5d(&tmY, src + s * 16384, bc0, w, h, bt, tc.b);
            }
          }
          ptx::bulk_commit();
        }
      }
    } else if (interior) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int cg = tc.n0 + 8 * j + cpair;
        const int n_il = p.up_time == 2 ? cg / chalf : 0;
        const int cc = cg - n_il * chalf;
        const int t_o = p.up_time == 2 ? 2 * tc.t + n_il - 1 : tc.t;
        const bool tok = t_o >= 0;
        const long long coff = t_o * p.ys_t + cc * p.ys_c;
        const float b0 = p.bias ? __ldg(p.bias + cg) : 0.f, b1 = p.bias ? __ldg(p.bias + cg + 1) : 0.f;
        float gs0 = 0.f, gq0 = 0.f, gs1 = 0.f, gq1 = 0.f;
        if (tok) {
#pragma unroll
          for (int s = 0; s < kMaxAcc; ++s) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              float a0 = fmaf(acc[s][4 * j + 2 * rr], p.alpha, b0);
              float a1 = fmaf(acc[s][4 * j + 2 * rr + 1], p.alpha, b1);
              const long long off = roff[s][rr] + coff;
              if (p.residual) {
                const float2 rf = E::to_f2(__ldg(reinterpret_cast<const typename E::P*>(reinterpret_cast<const T*>(p.residual) + off)));
                a0 += rf.x;
                a1 += rf.y;
              }
              const typename E::P o = E::pack2(a0, a1);
              *reinterpret_cast<typename E::P*>(reinterpret_cast<T*>(p.y) + off) = o;
              const float2 of = E::to_f2(o);
              gs0 += of.x;
              gq0 = fmaf(of.x, of.x, gq0);
              gs1 += of.y;
              gq1 = fmaf(of.y, of.y, gq1);
            }
          }
        }
        if (p.gn_stats) gn_add(gs0, gq0, gs1, gq1, cc, tok, true);
      }
    } else {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (tc.n0 + 8 * j >= p.Cout) break;   // warp-uniform
        const int cg = tc.n0 + 8 * j + cpair;
        const bool c0ok = cg < p.Cout, c1ok = cg + 1 < p.Cout;
        // output coordinates (time interleave of Upsample3D folded in); Cout is even with up_time, so cg and cg + 1
        // land in the same half
        const int n_il = p.up_time == 2 ? cg / chalf : 0;
        const int cc = cg - n_il * chalf;
        const int t_o = p.up_time == 2 ? 2 * tc.t + n_il - 1 : tc.t;
        const bool tok = t_o >= 0 && c0ok;
        const long long coff = t_o * p.ys_t + cc * p.ys_c;
        float b0 = 0.f, b1 = 0.f;
        if (p.bias && !bias_m) {
          if (c0ok) b0 = __ldg(p.bias + cg);
          if (c1ok) b1 = __ldg(p.bias + cg + 1);
        }
        float gs0 = 0.f, gq0 = 0.f, gs1 = 0.f, gq1 = 0.f;
#pragma unroll
        for (int s = 0; s < kMaxAcc; ++s) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            if (!rok[s][rr] || !tok) continue;
            const float bb0 = bias_m ? rbias[s][rr] : b0, bb1 = bias_m ? rbias[s][rr] : b1;
            float a0 = fmaf(acc[s][4 * j + 2 * rr], p.alpha, bb0);
            float a1 = fmaf(acc[s][4 * j + 2 * rr + 1], p.alpha, bb1);
            const long long off = roff[s][rr] + coff;
            if (out_f32) {
              // fp32 logits (S = q k^T): no residual, no interleave
              float* yf = reinterpret_cast<float*>(p.y) + off;
              if (p.vec2 && c1ok) {
                *reinterpret_cast<float2*>(yf) = make_float2(a0, a1);
              } else {
                yf[0] = a0;
                if (c1ok) yf[p.ys_c] = a1;
              }
              continue;
            }
            T* yp = reinterpret_cast<T*>(p.y) + off;
            const T* rp = p.residual ? reinterpret_cast<const T*>(p.residual) + off : nullptr;
            if (p.vec2 && c1ok) {
              if (rp) {
                const float2 rf = E::to_f2(__ldg(reinterpret_cast<const typename E::P*>(rp)));
                a0 += rf.x;
                a1 += rf.y;
              }
              const typename E::P o = E::pack2(a0, a1);
              *reinterpret_cast<typename E::P*>(yp) = o;
              const float2 of = E::to_f2(o);
              a0 = of.x;
              a1 = of.y;
            } else {
              if (rp) {
                a0 += E::to_f(rp[0]);
                if (c1ok) a1 += E::to_f(rp[p.ys_c]);
              }
              const T o0 = E::from_f(a0), o1 = E::from_f(a1);
              yp[0] = o0;
              if (c1ok) yp[p.ys_c] = o1;
              a0 = E::to_f(o0);
              a1 = E::to_f(o1);
            }
            // GroupNorm statistics of the consumer, from the stored (rounded) values
            gs0 += a0;
            gq0 = fmaf(a0, a0, gq0);
            if (c1ok) {
              gs1 += a1;
              gq1 = fmaf(a1, a1, gq1);
            }
          }
        }
        if (p.gn_stats) gn_add(gs0, gq0, gs1, gq1, cc, tok, c1ok);
      }
    }
  }

  if (traced && threadIdx.x == 128) trc[6] = ptx::globaltimer_ns();
  if (p.gn_stats) {
    ptx::named_bar_sync(1, 256);   // both MMA warpgroups' bins are in
    const int ct = static_cast<int>(threadIdx.x) - 128;
    if (ct < 2 * p.gn_groups) {
      const unsigned long long vsum = gn_bins[ct];
      if (vsum != 0ull)
        atomicAdd(reinterpret_cast<unsigned long long*>(p.gn_stats) + static_cast<size_t>(tc.b) * 2 * p.gn_groups + ct, vsum);
    }
  }
  // the staged tile must stay in shared memory until the TMA unit has read it (not until the global writes land)
  if (kCB == 64 && p.tma_epi && wg_leader) ptx::bulk_wait_read<0>();
  if (traced && threadIdx.x == 128) {
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    trc[7] = (ptx::globaltimer_ns() & 0xFFFFFFFFFFFFull) | (static_cast<unsigned long long>(smid) << 48);
  }
}

// ---------------------------------------------------------------------------------------- host side
// cuTensorMapEncodeTiled is a pure function of its arguments and costs 1-2 us on the host; a network pass issues the same
// few hundred (pointer, shape) combinations call after call (the activation buffers come back from the caching allocator at
// the same addresses), so the encoded maps are memoised per thread, keyed by the full argument list (SURVEY 8b: "optional
// descriptor cache keyed by (ptr, shape)").
struct TmapKey {
  const void* ptr;
  uint32_t rank, swizzle, esz;
  cuuint64_t dims[5], strides[4];
  cuuint32_t box[5], estr[5];
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapSlot {
  TmapKey key;
  CUtensorMap map;
  bool valid;
};
static constexpr int kTmapSlots = 1024;

// Element size of an activation dtype in bytes, and channels per 128-byte operand row.
static int elem_bytes(int dtype) { return dtype == CVVAE_F32 ? 4 : 2; }
static int chan_block(int dtype) { return 128 / elem_bytes(dtype); }

static bool encode_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_b,
                       const cuuint32_t* box, const cuuint32_t* estr, int esz,
                       CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  static thread_local TmapSlot* cache = nullptr;
  if (!cache) cache = static_cast<TmapSlot*>(calloc(kTmapSlots, sizeof(TmapSlot)));
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = ptr;
  key.rank = static_cast<uint32_t>(rank);
  key.swizzle = static_cast<uint32_t>(swizzle);
  key.esz = static_cast<uint32_t>(esz);
  for (int i = 0; i < rank; ++i) {
    key.dims[i] = dims[i];
    key.box[i] = box[i];
    key.estr[i] = estr[i];
    if (i + 1 < rank) key.strides[i] = strides_b[i];
  }
  uint64_t h = 1469598103934665603ull;  // FNV-1a over the key bytes
  const unsigned char* kb = reinterpret_cast<const unsigned char*>(&key);
  for (size_t i = 0; i < sizeof(key); ++i) h = (h ^ kb[i]) * 1099511628211ull;
  TmapSlot* slot = cache ? &cache[h % kTmapSlots] : nullptr;
  if (slot && slot->valid && slot->key == key) {
    *m = slot->map;
    return true;
  }
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return false;
  }
  CUresult r = enc(m, esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, rank, const_cast<void*>(ptr), dims, strides_b, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
              (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
              rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
    return false;
  }
  if (slot) {
    slot->key = key;
    slot->map = *m;
    slot->valid = true;
  }
  return true;
}

bool conv_tc_eligible(const cvvae_conv_desc* d, const char** why) {
  const cvvae_tensor5& x = d->x;
  auto fail = [&](const char* m) {
    if (why) *why = m;
    return false;
  };
  if (x.s_c != 1) return fail("input channel stride != 1");
  if (d->w_ld % 8 != 0 || (d->w_ld == 0 && x.C % 8 != 0)) return fail("weight row stride not a 16-byte multiple");
  if ((x.s_w % 8) || (x.s_h % 8) || (x.s_t % 8) || (x.s_b % 8)) return fail("input strides not 16-byte multiples");
  if (reinterpret_cast<uintptr_t>(x.ptr) % 16) return fail("input pointer not 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d->w) % 16) return fail("weight pointer not 16-byte aligned");
  if (d->pad_hw != CVVAE_PAD_ZERO) {
    // replicate padding in H/W is only needed when a tap can actually leave the image
    const int lo_h = d->off_h, hi_h = (d->y.H - 1) * d->sh + d->KH - 1 + d->off_h;
    const int lo_w = d->off_w, hi_w = (d->y.W - 1) * d->sw + d->KW - 1 + d->off_w;
    if (lo_h < 0 || lo_w < 0 || hi_h >= x.H || hi_w >= x.W) return fail("replicate H/W padding needs a pre-padded input");
  }
  if (d->sh > 2 || d->sw > 2 || d->sh != d->sw) return fail("unsupported spatial stride");
  if (d->KH > 3 || d->KW > 3 || d->KT > 3) return fail("kernel extent > 3");
  if (d->up_time == 2 && (d->Cout % 2)) return fail("odd Cout with up_time");
  return true;
}

static unsigned long long* g_trace_buf = nullptr;
static int g_trace_n = 0;
void conv_tc_set_trace(unsigned long long* buf, int n) {
  g_trace_buf = buf;
  g_trace_n = n;
}

template <int DT, int BN>
static int launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmA2, const CUtensorMap& tmB2,
                     const CUtensorMap& tmY, const CUtensorMap& tmR, const ConvTcParams& p, unsigned grid, size_t smem,
                     cudaStream_t stream) {
  static PerDeviceOnce attr_set;   // the > 48 KB shared-memory opt-in is per device
  if (attr_set.need()) {
    CVVAE_CUDA(cudaFuncSetAttribute(conv_tc_kernel<DT, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_set.mark();
  }
  conv_tc_kernel<DT, BN><<<grid, kThreads, smem, stream>>>(tmA, tmB, tmA2, tmB2, tmY, tmR, p);
  return CVVAE_OK;
}

// Byte strides of y's W, H, T and B axes for a tensor map, or false when TMA cannot address y: channel stride != 1, or a
// pointer or stride that is not a multiple of 16 bytes.  An axis of extent 1 may carry any stride; it gets a valid one.
static bool y_map_strides(const cvvae_tensor5& y, int esz, cuuint64_t* strides) {
  const long long s[4] = {y.s_w, y.s_h, y.s_t, y.s_b};
  const int n[4] = {y.W, y.H, y.T, y.B};
  if (y.s_c != 1 || reinterpret_cast<uintptr_t>(y.ptr) % 16) return false;
  for (int i = 0; i < 4; ++i) {
    if (n[i] == 1) {
      strides[i] = (static_cast<cuuint64_t>(y.C) * esz + 15) & ~cuuint64_t(15);
    } else {
      if (s[i] <= 0 || (s[i] * esz) % 16) return false;
      strides[i] = static_cast<cuuint64_t>(s[i]) * esz;
    }
  }
  return true;
}

// The output goes through shared memory and TMA stores (and the residual comes in by TMA) when y is a 16-bit channels-last
// tensor TMA can address, with the residual on the same strides and a block of 64 channels staged per A-ring slot (the
// BN / 64 blocks need that many slots; a slot always holds one, since slab_rows >= TH).  fp32 outputs (logits, fp32
// models), bias along M and the NCDHW / unaligned views keep the register epilogue, as does CVVAE_TMA_EPILOGUE=0.
static bool tma_epilogue_ok(const cvvae_conv_desc* d, const ConvTcParams& p) {
  const char* env = getenv("CVVAE_TMA_EPILOGUE");
  if (env && strcmp(env, "0") == 0) return false;
  if (d->dtype == CVVAE_F32 || (d->flags & (CVVAE_CONV_OUT_F32 | CVVAE_CONV_BIAS_ALONG_M))) return false;
  cuuint64_t strides[4];
  if (!y_map_strides(d->y, 2, strides)) return false;
  if (d->residual && reinterpret_cast<uintptr_t>(d->residual) % 16) return false;
  if (p.Cout % 8 || (p.up_time == 2 && (p.Cout / 2) % 64)) return false;
  return p.N_cta / 64 <= p.NA;
}

// The launch plan of a descriptor: geometry, epilogue pointers and strides, tiling (N_cta, NACC, TW / TH, tile counts),
// operand ring depths, dynamic shared memory and grid.  conv_tc_launch runs exactly this plan and cvvae_conv_tc_plan
// reports it, so a test can check which plan it ran.  The fused shortcut, GroupNorm and trace fields are the launch's.
static int conv_tc_plan(const cvvae_conv_desc* d, ConvTcParams& p, size_t& smem, long long& grid) {
  const char* why = nullptr;
  if (!conv_tc_eligible(d, &why)) {
    set_error("cvvae_conv3d_tc: not eligible: %s", why);
    return CVVAE_E_UNSUPPORTED;
  }
  const cvvae_tensor5& x = d->x;
  const cvvae_tensor5& y = d->y;
  p = ConvTcParams{};
  p.B = x.B;
  p.T_in = x.T;
  p.Cin = x.C;
  p.Cout = d->Cout;
  p.up_time = d->up_time == 2 ? 2 : 1;
  p.T_out = p.up_time == 2 ? (y.T + 1) / 2 : y.T;
  p.H_out = y.H;
  p.W_out = y.W;
  p.KT = d->KT; p.KH = d->KH; p.KW = d->KW;
  p.st = d->st; p.sh = d->sh; p.sw = d->sw;
  p.off_t = d->off_t; p.off_h = d->off_h; p.off_w = d->off_w;
  p.pad_t = d->pad_t;
  p.flags = d->flags;
  p.alpha = d->alpha;
  p.bias = d->bias;
  p.residual = d->residual;
  p.y = y.ptr;
  p.ys_b = y.s_b; p.ys_t = y.s_t; p.ys_h = y.s_h; p.ys_w = y.s_w; p.ys_c = y.s_c;
  p.yC = y.C;
  if (d->flags & CVVAE_CONV_X_SHARED) CVVAE_CHECK_ARG(x.B == 1, "conv: CVVAE_CONV_X_SHARED needs x.B == 1");
  else CVVAE_CHECK_ARG(y.B == x.B, "conv: batch mismatch");
  if (d->flags & CVVAE_CONV_W_PER_BATCH)
    CVVAE_CHECK_ARG(d->KT * d->KH * d->KW == 1 && p.up_time == 1 && !d->gn_stats, "conv: per-batch weights need a 1x1x1 problem");
  p.B = y.B;
  CVVAE_CHECK_ARG(y.C == (p.up_time == 2 ? d->Cout / 2 : d->Cout), "conv: y.C %d inconsistent with Cout %d / up_time %d",
                  y.C, d->Cout, p.up_time);
  // channel pairs as one word: unit channel stride, even position strides, word-aligned pointers
  {
    const bool out_f32 = (d->flags & CVVAE_CONV_OUT_F32) != 0;
    const uintptr_t align = (out_f32 || d->dtype == CVVAE_F32) ? 8 : 4;
    p.vec2 = (y.s_c == 1) && !(y.s_w % 2) && !(y.s_h % 2) && !(y.s_t % 2) && !(y.s_b % 2) &&
             (reinterpret_cast<uintptr_t>(y.ptr) % align == 0) &&
             (!d->residual || reinterpret_cast<uintptr_t>(d->residual) % align == 0);
  }
  if (d->flags & CVVAE_CONV_OUT_F32)
    CVVAE_CHECK_ARG(!d->residual && p.up_time == 1, "conv: fp32 output excludes residual / up_time");

  // ---- tiling: BN output channels per CTA, NACC 128-position sub-tiles (two 64-row halves, one per MMA warpgroup)
  const int N_cta = p.Cout >= 256 ? 256 : (p.Cout > 64 ? 128 : 64);
  p.N_cta = N_cta;
  p.n_tiles_n = (p.Cout + N_cta - 1) / N_cta;
  p.NACC = 256 / N_cta;   // 64 x N_cta x NACC fp32 per warpgroup = 128 accumulator registers per thread
  p.flat = (p.H_out == 1 && d->KH == 1 && d->KW == 1 && d->sw == 1 && d->sh == 1 && x.H == 1) ? 1 : 0;
  if (d->flags & (CVVAE_CONV_W_PER_BATCH | CVVAE_CONV_X_SHARED))
    CVVAE_CHECK_ARG(p.flat, "conv: batched-GEMM flags need a flat problem (H == 1, 1x1x1, stride 1)");
  const int cb = chan_block(d->dtype);
  p.cblocks = (p.Cin + cb - 1) / cb;
  for (;;) {
    if (p.flat) {
      p.TW = 128; p.ROWS = 1; p.TH = 1;
      p.KHs = 1; p.n_hgroups = 1; p.slab_rows = p.NACC;
      p.tiles_w = (p.W_out + p.NACC * 128 - 1) / (p.NACC * 128);
      p.tiles_h = 1;
    } else {
      p.KHs = (d->sh == 1) ? d->KH : 1;
      p.n_hgroups = d->KH / p.KHs;
      long long best_cost = -1;
      int best_tw = 16;
      for (int tw = 8; tw <= 128; tw *= 2) {
        const int rows = 128 / tw;
        const int th = rows * p.NACC;
        if (tw * d->sw > 256 || (th + p.KHs - 1) * d->sh > 256) continue;
        const long long tiles_w = (p.W_out + tw - 1) / tw;
        const long long subtiles_h = (p.H_out + rows - 1) / rows;
        const long long tiles_h = (p.H_out + th - 1) / th;
        // MMA work ~ sub-tiles; slab traffic ~ (th + halo) rows per tile
        const long long cost = tiles_w * subtiles_h * 128 * 16 + tiles_w * tiles_h * (th + p.KHs - 1) * tw * 3;
        if (best_cost < 0 || cost < best_cost) {
          best_cost = cost;
          best_tw = tw;
        }
      }
      p.TW = best_tw;
      p.ROWS = 128 / p.TW;
      p.TH = p.ROWS * p.NACC;
      p.slab_rows = p.TH + p.KHs - 1;
      p.tiles_w = (p.W_out + p.TW - 1) / p.TW;
      p.tiles_h = (p.H_out + p.TH - 1) / p.TH;
    }
    // small problems (latent-resolution layers, single images, attention GEMMs): fewer sub-tiles per CTA = more CTAs.
    // The count is per SAMPLE so that the plan - hence every rounding - is independent of the batch size.
    const long long ctas_per_sample = 1ll * p.n_tiles_n * p.T_out * p.tiles_w * p.tiles_h;
    if (p.NACC <= 1 || ctas_per_sample >= num_sms()) break;
    p.NACC /= 2;
  }
  p.slab_bytes = p.flat ? static_cast<uint32_t>(p.NACC) * 16384u : static_cast<uint32_t>(p.slab_rows * p.TW) * 128u;
  p.slab_stride = (p.slab_bytes + 1023u) & ~1023u;
  p.b_bytes = static_cast<uint32_t>(N_cta) * 128u;

  // ---- shared memory budget: 227 KB - alignment slack - barriers
  const size_t budget = 232448 - 1024 - kBarBytes;
  int NB = 4;
  while (NB > 2 && static_cast<size_t>(NB) * p.b_bytes + 2ull * p.slab_stride > budget) --NB;
  const size_t rest = budget - static_cast<size_t>(NB) * p.b_bytes;
  int NA = static_cast<int>(rest / p.slab_stride);
  if (NA > 4) NA = 4;
  CVVAE_CHECK_ARG(NA >= 2, "conv_tc: slab of %u bytes does not fit the shared-memory budget", p.slab_bytes);
  // spend what is left on more weight stages
  while (NB < 8 && static_cast<size_t>(NB + 1) * p.b_bytes + static_cast<size_t>(NA) * p.slab_stride <= budget) ++NB;
  p.NA = NA;
  p.NB = NB;
  smem = 1024 + static_cast<size_t>(NA) * p.slab_stride + static_cast<size_t>(NB) * p.b_bytes + kBarBytes;
  p.tma_epi = tma_epilogue_ok(d, p) ? 1 : 0;

  grid = 1ll * p.n_tiles_n * p.T_out * p.tiles_w * p.tiles_h * p.B;
  CVVAE_CHECK_ARG(grid > 0 && grid < (1ll << 31), "conv_tc: grid size %lld out of range", grid);
  return CVVAE_OK;
}

int conv_tc_launch(const cvvae_conv_desc* d, cudaStream_t stream) {
  ConvTcParams p;
  size_t smem = 0;
  long long grid = 0;
  const int prc = conv_tc_plan(d, p, smem, grid);
  if (prc != CVVAE_OK) return prc;
  const cvvae_tensor5& x = d->x;
  const cvvae_tensor5& y = d->y;
  const int N_cta = p.N_cta;
  const int esz = elem_bytes(d->dtype);
  const int cb = chan_block(d->dtype);
  p.trace = g_trace_buf;
  p.trace_n = g_trace_n;

  // ---- tensor maps
  CUtensorMap tmA, tmB;
  {
    cuuint64_t dims[5] = {(cuuint64_t)x.C, (cuuint64_t)x.W, (cuuint64_t)x.H, (cuuint64_t)x.T, (cuuint64_t)x.B};
    cuuint64_t strides[4] = {(cuuint64_t)x.s_w * esz, (cuuint64_t)x.s_h * esz, (cuuint64_t)x.s_t * esz, (cuuint64_t)x.s_b * esz};
    // degenerate dims may carry meaningless strides; TMA wants multiples of 16 and monotone-ish validity
    for (int i = 0; i < 4; ++i)
      if (dims[i + 1] == 1 && (strides[i] == 0 || strides[i] % 16)) strides[i] = (cuuint64_t)x.C * esz;
    cuuint32_t box[5], estr[5] = {1, (cuuint32_t)d->sw, (cuuint32_t)d->sh, 1, 1};
    box[0] = (cuuint32_t)cb;
    if (p.flat) {
      box[1] = 128; box[2] = 1;
    } else {
      box[1] = (cuuint32_t)(p.TW * d->sw);
      box[2] = (cuuint32_t)(p.slab_rows * d->sh);
    }
    box[3] = 1; box[4] = 1;
    if (!encode_map(&tmA, x.ptr, 5, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
  }
  {
    const int taps = (d->flags & CVVAE_CONV_W_PER_BATCH) ? x.B > y.B ? x.B : y.B : d->KT * d->KH * d->KW;
    cuuint64_t dims[3] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Cout, (cuuint64_t)taps};
    const cuuint64_t wld = d->w_ld ? (cuuint64_t)d->w_ld : (cuuint64_t)p.Cin;
    cuuint64_t strides[2] = {wld * esz, wld * p.Cout * esz};
    cuuint32_t box[3] = {(cuuint32_t)cb, (cuuint32_t)N_cta, 1}, estr[3] = {1, 1, 1};
    if (!encode_map(&tmB, d->w, 3, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
  }

  // ---- fused 1x1 shortcut: a second input tensor (same positions as the output) and a [Cout][Cin2] matrix
  CUtensorMap tmA2 = tmA, tmB2 = tmB;
  p.Cin2 = 0;
  p.cblocks2 = 0;
  if (d->w2) {
    const cvvae_tensor5& x2 = d->x2;
    CVVAE_CHECK_ARG(tensor_ok(&x2) && x2.B == y.B && x2.T == y.T && x2.H == y.H && x2.W == y.W,
                    "conv: fused shortcut input must have the output's [B,T,H,W] extents");
    CVVAE_CHECK_ARG(x2.s_c == 1 && x2.C % 8 == 0 && !(x2.s_w % 8) && !(x2.s_h % 8) && !(x2.s_t % 8) && !(x2.s_b % 8) &&
                        reinterpret_cast<uintptr_t>(x2.ptr) % 16 == 0 && reinterpret_cast<uintptr_t>(d->w2) % 16 == 0,
                    "conv: fused shortcut operands must be 16-byte aligned channels-last views with C %% 8 == 0");
    CVVAE_CHECK_ARG(!p.flat && p.up_time == 1 && d->st == 1 && d->sh == 1 && d->sw == 1 && !d->residual &&
                        !(d->flags & (CVVAE_CONV_BIAS_ALONG_M | CVVAE_CONV_OUT_F32 | CVVAE_CONV_W_PER_BATCH | CVVAE_CONV_X_SHARED)),
                    "conv: a fused shortcut needs a stride-1 spatial convolution without residual / interleave");
    CVVAE_CHECK_ARG(-d->off_h >= 0 && -d->off_h < d->KH && -d->off_w >= 0 && -d->off_w < d->KW && d->off_t <= 0 && -d->off_t < d->KT,
                    "conv: fused shortcut needs the centre tap inside the kernel window");
    p.Cin2 = x2.C;
    p.cblocks2 = (x2.C + cb - 1) / cb;
    {
      cuuint64_t dims[5] = {(cuuint64_t)x2.C, (cuuint64_t)x2.W, (cuuint64_t)x2.H, (cuuint64_t)x2.T, (cuuint64_t)x2.B};
      cuuint64_t strides[4] = {(cuuint64_t)x2.s_w * esz, (cuuint64_t)x2.s_h * esz, (cuuint64_t)x2.s_t * esz, (cuuint64_t)x2.s_b * esz};
      for (int i = 0; i < 4; ++i)
        if (dims[i + 1] == 1 && (strides[i] == 0 || strides[i] % 16)) strides[i] = (cuuint64_t)x2.C * esz;
      cuuint32_t box[5] = {(cuuint32_t)cb, (cuuint32_t)p.TW, (cuuint32_t)p.slab_rows, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
      if (!encode_map(&tmA2, x2.ptr, 5, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
    }
    {
      cuuint64_t dims[3] = {(cuuint64_t)x2.C, (cuuint64_t)p.Cout, 1};
      cuuint64_t strides[2] = {(cuuint64_t)x2.C * esz, (cuuint64_t)x2.C * p.Cout * esz};
      cuuint32_t box[3] = {(cuuint32_t)cb, (cuuint32_t)N_cta, 1}, estr[3] = {1, 1, 1};
      if (!encode_map(&tmB2, d->w2, 3, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
    }
  }

  // fused GroupNorm statistics need power-of-two channels per group and one sample per CTA index
  p.gn_stats = nullptr;
  if (d->gn_stats) {
    const int cpg = d->gn_groups > 0 ? y.C / d->gn_groups : 0;
    const bool ok = !(d->flags & CVVAE_CONV_OUT_F32) && d->gn_groups > 0 && d->gn_groups <= 64 && y.C % d->gn_groups == 0 &&
                    cpg >= 1 && (cpg & (cpg - 1)) == 0;
    if (!ok) {
      set_error("conv_tc: fused GroupNorm statistics unsupported for this output (C=%d groups=%d)", y.C, d->gn_groups);
      return CVVAE_E_UNSUPPORTED;
    }
    p.gn_stats = d->gn_stats;
    p.gn_groups = d->gn_groups;
    p.gn_cpg = cpg;
  }

  // ---- TMA epilogue: y and the residual (same strides) as 5-D maps, one box = 64 positions x 64 channels
  CUtensorMap tmY = tmA, tmR = tmA;
  if (p.tma_epi) {
    cuuint64_t dims[5] = {(cuuint64_t)y.C, (cuuint64_t)y.W, (cuuint64_t)y.H, (cuuint64_t)y.T, (cuuint64_t)y.B};
    cuuint64_t strides[4];
    y_map_strides(y, esz, strides);
    const bool rows = p.ROWS >= 2;
    cuuint32_t box[5] = {(cuuint32_t)cb, (cuuint32_t)(rows ? p.TW : 64), (cuuint32_t)(rows ? p.ROWS / 2 : 1), 1, 1},
               estr[5] = {1, 1, 1, 1, 1};
    if (!encode_map(&tmY, y.ptr, 5, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
    if (d->residual && !encode_map(&tmR, d->residual, 5, dims, strides, box, estr, esz)) return CVVAE_E_CUDA;
  }

  int rc = CVVAE_OK;
  CVVAE_DISPATCH_DTYPE(d->dtype, {
    if (N_cta == 256) rc = launch_bn<DT, 256>(tmA, tmB, tmA2, tmB2, tmY, tmR, p, static_cast<unsigned>(grid), smem, stream);
    else if (N_cta == 128) rc = launch_bn<DT, 128>(tmA, tmB, tmA2, tmB2, tmY, tmR, p, static_cast<unsigned>(grid), smem, stream);
    else rc = launch_bn<DT, 64>(tmA, tmB, tmA2, tmB2, tmY, tmR, p, static_cast<unsigned>(grid), smem, stream);
  });
  if (rc != CVVAE_OK) return rc;
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}

static int conv_tc_plan_query(const cvvae_conv_desc* d, int32_t* out, int32_t n) {
  ConvTcParams p;
  size_t smem = 0;
  long long grid = 0;
  const int rc = conv_tc_plan(d, p, smem, grid);
  if (rc != CVVAE_OK && rc != CVVAE_E_UNSUPPORTED) return rc;
  const bool ok = rc == CVVAE_OK;
  const int32_t v[] = {ok ? 1 : 0,
                       ok ? p.N_cta : 0,
                       ok ? p.NACC : 0,
                       ok ? p.TW : 0,
                       ok ? p.ROWS : 0,
                       ok ? p.TH : 0,
                       ok ? p.tiles_w : 0,
                       ok ? p.tiles_h : 0,
                       ok ? p.n_tiles_n : 0,
                       ok ? p.flat : 0,
                       ok ? p.NA : 0,
                       ok ? p.NB : 0,
                       ok ? static_cast<int32_t>(grid) : 0,
                       ok ? p.vec2 : 0,
                       ok ? p.tma_epi : 0};
  constexpr int32_t kFields = static_cast<int32_t>(sizeof(v) / sizeof(v[0]));
  for (int32_t i = 0; i < n && i < kFields; ++i) out[i] = v[i];
  return kFields;
}

}  // namespace cvvae

extern "C" int cvvae_conv_tc_set_trace(void* device_buf, int32_t n_ctas) {
  cvvae::conv_tc_set_trace(static_cast<unsigned long long*>(device_buf), device_buf ? n_ctas : 0);
  return CVVAE_OK;
}

extern "C" int cvvae_conv_tc_plan(const cvvae_conv_desc* d, int32_t* out, int32_t n) {
  CVVAE_CHECK_ARG(d && cvvae::tensor_ok(&d->x) && cvvae::tensor_ok(&d->y) && d->w && (out || n <= 0),
                  "cvvae_conv_tc_plan: null argument");
  return cvvae::conv_tc_plan_query(d, out, n);
}

extern "C" int cvvae_conv3d_tc(const cvvae_conv_desc* d, void* stream) {
  CVVAE_CHECK_ARG(d && cvvae::tensor_ok(&d->x) && cvvae::tensor_ok(&d->y) && d->w, "cvvae_conv3d_tc: null argument");
  return cvvae::conv_tc_launch(d, static_cast<cudaStream_t>(stream));
}
