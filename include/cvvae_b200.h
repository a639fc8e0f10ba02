/*
 * cvvae_b200 - C ABI of the H100-native (sm_90a) CV-VAE encode()/decode() hot path.
 *
 * The reference (AILab-CVC/CV-VAE) is pure Python on PyTorch and has no FFI of its own; the seam this
 * library replaces is the `nn.Module.__call__` operator boundary inside `self.encoder(x)` /
 * `self.decoder(z)` (models/modeling_vae.py:162,249), i.e. the PyTorch library ops listed below.  A
 * reference-side binding is a ctypes stub that passes `tensor.data_ptr()` and the current CUDA stream
 * (see INTEGRATION.md).
 *
 * Conventions
 *   - every entry point returns 0 on success, a negative CVVAE_E_* code otherwise; the message of the
 *     last failure on the calling thread is available from cvvae_last_error().  Nothing aborts or throws.
 *   - no allocation inside: the caller owns inputs, outputs and workspaces (device pointers).
 *   - every call is asynchronous on the `stream` it is given (a cudaStream_t passed as void*).
 *   - activations are channels-last: element (b,t,h,w,c) lives at b*s_b + t*s_t + h*s_h + w*s_w + c*s_c
 *     (strides in ELEMENTS).  The tensor-core path needs s_c == 1 on its input.
 *   - dtype: CVVAE_F16, CVVAE_BF16 or CVVAE_F32 for activations and packed weights; bias / norm parameters are fp32;
 *     GroupNorm statistics are 64-bit fixed point (order-independent integer accumulation, see below).
 *     CVVAE_F32: activations and packed weights are fp32 and the tensor-core path multiplies in TF32 (10-bit mantissa
 *     products, fp32 accumulation), as PyTorch's default fp32 convolution does on this GPU.  Outputs whose only
 *     consumers are tensor-core products (packed weights, GroupNorm / LayerNorm / softmax outputs, pack_taps_hw and the
 *     channels-first -> channels-last copy of a network input) are stored rounded to the nearest TF32 value; every other output
 *     (convolution outputs: residual stream, q / k / v, attention output) is full fp32.  The video_io entry points and
 *     cvvae_conv3d_stacked are 16-bit only and reject CVVAE_F32.
 */
#ifndef CVVAE_B200_H_
#define CVVAE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CVVAE_ABI_VERSION 3

enum { CVVAE_F16 = 0, CVVAE_BF16 = 1, CVVAE_F32 = 2 };
enum { CVVAE_PAD_ZERO = 0, CVVAE_PAD_REPLICATE = 1 };
enum {
  CVVAE_OK = 0,
  CVVAE_E_ARG = -1,      /* invalid / unsupported argument combination */
  CVVAE_E_CUDA = -2,     /* CUDA runtime / driver error                */
  CVVAE_E_UNSUPPORTED = -3
};
enum {
  CVVAE_CONV_BIAS_ALONG_M = 1, /* bias indexed by flattened output position instead of channel */
  CVVAE_CONV_FORCE_DIRECT = 2, /* debugging: route cvvae_conv3d() to the CUDA-core kernel       */
  CVVAE_CONV_OUT_F32 = 4,      /* y holds fp32 (strides in fp32 elements); no residual, up_time 1  */
  /* Batched GEMM over the B axis (the per-frame attention products, models/vae_models.py:446-461,500-528): */
  CVVAE_CONV_W_PER_BATCH = 8,  /* `w` holds one [Cout][Cin(ld)] matrix PER batch item ([y.B][Cout][w_ld], contiguous);
                                  1x1x1 flat problems only.  A CVVAE_CONV_BIAS_ALONG_M bias is then [T*H*W], shared  */
  CVVAE_CONV_X_SHARED = 16     /* x.B == 1: the same left operand for every batch item of y                       */
};

/* One strided channels-last 5-D tensor view. */
typedef struct cvvae_tensor5 {
  void* ptr;
  int32_t B, T, H, W, C;
  int64_t s_b, s_t, s_h, s_w, s_c; /* element strides */
} cvvae_tensor5;

/*
 * Convolution (3-D, per-frame 2-D as KT=1, 1x1x1, strided, and plain GEMM as a 1x1x1 conv).
 *
 * Replaces, in the reference:
 *   CausalConv3d.forward                models/vae_models.py:298-328, models/vae_blocks3d_sd3.py:81-104
 *   nn.Conv3d / Conv3d(replicate)       models/vae_models.py:361,953,  models/vae_blocks3d_sd3.py:16-46
 *   Conv2dWithExtraDim.forward          models/vae_models.py:331-340
 *   Downsample3D.forward                models/vae_models.py:251-263,  models/vae_blocks3d_sd3.py:224-239
 *   the conv + interleave of Upsample3D models/vae_models.py:229-232,  models/vae_blocks3d_sd3.py:352-362
 *   nin_shortcut / conv_shortcut, q/k/v/proj_out 1x1 convs and the Linear layers of the attention blocks.
 *
 * y[b, to, ho, wo, co] = alpha * ( sum_{kt,kh,kw,ci} x[b, ti, hi, wi, ci] * w[(kt,kh,kw), co, ci] )
 *                        + bias[co] + residual[b, to, ho, wo, co]
 *   ti = to*st + kt + off_t   (pad_t: ZERO -> taps outside [0,T) contribute 0; REPLICATE -> clamp)
 *   hi = ho*sh + kh + off_h, wi = wo*sw + kw + off_w  (pad_hw likewise)
 * With up_time == 2 (Upsample3D, "b (n c) t h w -> b c (t n) h w" then drop frame 0): output channel
 * co = n*(Cout/2) + c of conv-time t is stored at y[b, 2t+n-1, ho, wo, c] (dropped when 2t+n-1 < 0);
 * y.C == Cout/2 and y.T == 2*T_conv-1 in that case.
 * Weights are pre-packed by cvvae_pack_conv_weight(): [KT*KH*KW][Cout][Cin], Cin contiguous.
 */
typedef struct cvvae_conv_desc {
  cvvae_tensor5 x;          /* input  */
  cvvae_tensor5 y;          /* output (geometry after the optional time interleave) */
  const void* w;            /* packed weights, activation dtype */
  int64_t w_ld;             /* element stride between weight rows (0 -> Cin); multiple of 8 for the tc path */
  const float* bias;        /* [Cout] (or [B*T*H*W] with CVVAE_CONV_BIAS_ALONG_M), may be NULL */
  const void* residual;     /* same geometry/strides as y, may be NULL */
  int32_t Cout;             /* conv output channels (before interleave) */
  int32_t KT, KH, KW;
  int32_t st, sh, sw;
  int32_t off_t, off_h, off_w;
  int32_t pad_t, pad_hw;    /* CVVAE_PAD_* */
  int32_t up_time;          /* 1 or 2 */
  int32_t dtype;            /* CVVAE_F16 / CVVAE_BF16 / CVVAE_F32 */
  int32_t flags;            /* CVVAE_CONV_* */
  float alpha;
  int64_t* gn_stats;        /* optional [B][gn_groups][2] int64 fixed point as above (of the STORED y), accumulated:
                               GroupNorm statistics of the consumer, produced in the conv epilogue instead of a
                               separate pass over y.  The caller zeroes it (several launches may add to it).  */
  int32_t gn_groups;
  /* Optional fused 1x1 shortcut (ResnetBlock3D: `x = nin_shortcut(x); return x + h`, models/vae_models.py:386-388,406-410;
   * conv_shortcut of the sd3 blocks): y += sum_ci x2[b,t,h,w,ci] * w2[co][ci], accumulated in the same fp32 accumulators
   * as the taps (extra K steps), so the shortcut tensor is never written or re-read and the sum is rounded once.  x2 has
   * the OUTPUT's [B,T,H,W] extents (stride-1 'same' convolutions only), channels-last, C % 8 == 0; w2 is [Cout][x2.C] in the
   * activation dtype; `bias` then holds the sum of both biases.  w2 == NULL: none.  Tensor-core path only. */
  cvvae_tensor5 x2;
  const void* w2;
} cvvae_conv_desc;

/* Dispatcher: wgmma implicit-GEMM kernel when eligible (x.s_c==1, Cin%8==0, 16B-aligned strides,
 * pad_hw==ZERO), CUDA-core kernel otherwise (e.g. the 3/4-channel network inputs).              */
int cvvae_conv3d(const cvvae_conv_desc* d, void* stream);
int cvvae_conv3d_tc(const cvvae_conv_desc* d, void* stream);     /* tensor-core path only */
int cvvae_conv3d_direct(const cvvae_conv_desc* d, void* stream); /* CUDA-core path only   */
/* 1 if cvvae_conv3d() would take the tensor-core path for this descriptor, else 0. */
int cvvae_conv3d_is_tc(const cvvae_conv_desc* d);

/* Tap-stacked kernel for stride-1 (KT x) 3 x 3 convolutions with Cout <= 4 (Decoder.conv_out, 128 -> 3 at full
 * resolution; reference models/vae_models.py:942-944,999): the nine (kh,kw) taps are stacked along the MMA's N
 * dimension and the spatial shifts applied to the per-position partial sums afterwards.  Same descriptor as
 * cvvae_conv3d, except that `w` holds the STACKED weights [KT][80][Cin] (row (kh*3+kw)*8 + c, all other rows zero);
 * no residual / statistics / fp32 output.  pad_hw == REPLICATE needs a framed input (off_h = off_w = 0). */
int cvvae_conv3d_stacked(const cvvae_conv_desc* d, void* stream);

/* [Cout][Cin][KT][KH][KW] (PyTorch layout, contiguous, activation dtype) -> [KT*KH*KW][Cout][Cin].  CVVAE_F32: the packed
 * weights are rounded to the nearest TF32 value. */
int cvvae_pack_conv_weight(const void* w_oikkk, void* w_packed, int32_t Cout, int32_t Cin, int32_t taps,
                           int32_t dtype, void* stream);

/*
 * GroupNorm (+ optional SiLU), replacing Normalize()+nonlinearity (models/vae_models.py:187-195,
 * 392-401) and nn.GroupNorm+nn.SiLU of the sd3 blocks.  Statistics over (C/groups, T, H, W) per
 * sample; pass per_frame=1 for the attention blocks, whose GroupNorm sees T folded into the batch
 * (models/vae_models.py:466,533,622).
 *   stats workspace: int64 [B*(per_frame?T:1)][groups][2] FIXED POINT (sum * 2^20, sum of squares * 2^18): integer
 *   atomics make the accumulation order-independent, hence bit-reproducible; zeroed by cvvae_groupnorm_stats.
 */
int cvvae_groupnorm_stats(const cvvae_tensor5* x, int32_t groups, int32_t per_frame, int64_t* stats,
                          int32_t dtype, void* stream);
int cvvae_groupnorm_apply(const cvvae_tensor5* x, const cvvae_tensor5* y, int32_t groups, int32_t per_frame,
                          const int64_t* stats, const float* gamma, const float* beta, float eps,
                          int32_t silu, int32_t dtype, void* stream);

/* LayerNorm over C for every (b,t,h,w) token: norm_t of MemoryEfficientAttnVideoBlock
 * (models/vae_models.py:571,575). */
int cvvae_layernorm(const cvvae_tensor5* x, const cvvae_tensor5* y, const float* gamma, const float* beta,
                    float eps, int32_t dtype, void* stream);

/* Row softmax: fp32 logits s[rows][ld_s] -> probabilities p[rows][ld_p] in the activation dtype (first `cols` entries of
 * each row), fp32 math.  Part of softmax(q k^T / sqrt(C)) v (models/vae_models.py:456,518,607). */
int cvvae_softmax_rows(const float* s, int64_t ld_s, void* p, int64_t ld_p, int64_t rows, int32_t cols,
                       int32_t dtype, void* stream);

/* Temporal attention of MemoryEfficientAttnVideoBlock.attention_t (models/vae_models.py:573-587):
 * for every (b,h,w): tokens = the T frames, one head of dim C.  q,k,v,o are [B,T,H,W,C] views. */
int cvvae_attn_temporal(const cvvae_tensor5* q, const cvvae_tensor5* k, const cvvae_tensor5* v,
                        const cvvae_tensor5* o, int32_t dtype, void* stream);

/* Replicate the outermost valid row/column of the interior [1,H-1)x[1,W-1) into the 1-pixel frame of
 * a spatially pre-padded buffer (replicate padding of the sd3 convs, vae_blocks3d_sd3.py:87-98). */
int cvvae_replicate_border(const cvvae_tensor5* xpad, int32_t dtype, void* stream);

/* Generic strided copy / layout change between two 5-D views of equal logical shape; y may have more
 * channels than x, the extra channels are zero-filled (channel padding of the 3/4-channel network inputs).
 * CVVAE_F32: a copy from a channels-first view (x.s_c != 1) into a channels-last one (y.s_c == 1) is the gather of a
 * network input for its first convolution and stores values rounded to the nearest TF32; every other copy is exact. */
int cvvae_copy5(const cvvae_tensor5* x, const cvvae_tensor5* y, int32_t dtype, void* stream);

/* Spatial taps of a network-input convolution packed into channels (conv_in of Encoder / Decoder: 3 / 4 input channels,
 * models/vae_models.py:731-737, 877-883; vae_models3d_sd3.py:93-99): y[b,t,h,w,(kh*KW+kw)*x.C + c] =
 * x[b,t,h+kh+off_h,w+kw+off_w,c], zero (pad_hw = ZERO) or edge-clamped (REPLICATE) outside the image; channels of y beyond
 * KH*KW*x.C are zero.  x: any strides (the caller's NCDHW tensor); y: channels-last, C % 8 == 0, extents = the conv's
 * output extents in H and W.  The KT x KH x KW convolution then runs as KT x 1 x 1 over y with weights packed
 * [KT][Cout][y.C] in the same channel order. */
int cvvae_pack_taps_hw(const cvvae_tensor5* x, const cvvae_tensor5* y, int32_t KH, int32_t KW, int32_t off_h, int32_t off_w,
                       int32_t pad_hw, int32_t dtype, void* stream);

/* Tile blending, in place on b (models/modeling_vae.py:321-341):
 *   b[..., i] = (1 - i/ov) * a[..., La-ov+i] + (i/ov) * b[..., i]   for i in [0,ov) along axis
 * axis: 0 = width (blend_h), 1 = height (blend_v).  a and b are 5-D views with logical dims
 * [B,T,H,W,C] (any strides, e.g. NCDHW tensors described with s_c = T*H*W). */
int cvvae_blend(const cvvae_tensor5* a, const cvvae_tensor5* b, int32_t overlap, int32_t axis, int32_t dtype,
                void* stream);

/* Pixel pre/post-processing of the inference script, one pass each, bit-exact with the reference expressions:
 *   u8_to_f16:  uint8 frames [T,H,W,3] -> 16-bit [3,T,H,W] = frame.half() / 127.5 - 1.0   (cvvae_inference_video.py:30-38)
 *   f16_to_u8:  16-bit [3,T,H,W] -> uint8 [T,H,W,3] = ((clamp(x,-1,1) + 1.0) * 127.5).to(uint8)   (:47-50)
 * Both tensors are contiguous device buffers. */
int cvvae_video_u8_to_f16(const uint8_t* thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t dtype, void* stream);
int cvvae_video_f16_to_u8(const void* in_cthw, uint8_t* thwc, int32_t T, int32_t H, int32_t W, int32_t dtype, void* stream);
/* The script's `transforms.Resize(size=(height, width))` on the uint8 frames (cvvae_inference_video.py:15-17,28), on the GPU:
 * antialiased bilinear (triangle filter, support scaled by the down-scale factor, round half up), uint8 [T,H,W,3] ->
 * out_thwc uint8 [T,OH,OW,3] and/or out_cthw 16-bit [3,T,OH,OW] = resized.half() / 127.5 - 1.0 (either may be NULL).
 * fp32 arithmetic: within 1 LSB of torchvision's fixed-point uint8 path (differs on < 1 % of the pixels). */
int cvvae_video_resize_u8(const uint8_t* thwc, uint8_t* out_thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t OH,
                          int32_t OW, int32_t dtype, void* stream);

/* Diagnostics */
/* Per-CTA phase timestamps of the next conv_tc launches: device buffer of n_ctas x 8 uint64 (globaltimer ns:
 * entry, setup done, first A landed, first B landed, all MMAs issued, accumulators ready, epilogue done,
 * exit | smid<<48).  Pass NULL to switch off. */
int cvvae_conv_tc_set_trace(void* device_buf, int32_t n_ctas);
/* The tile plan cvvae_conv3d_tc() launches for this descriptor on the current device (it depends on the SM count), as
 * int32 values: eligible (0: the tensor-core path refuses it, reason in cvvae_last_error(), every other value 0), N_cta
 * (output channels per CTA), NACC (128-position sub-tiles per CTA), TW, ROWS (= 128/TW), TH (= ROWS*NACC; the patch of
 * one CTA is TH x TW positions, or NACC*128 positions along W when flat), tiles_w, tiles_h, n_tiles_n, flat, NA, NB
 * (activation / weight ring depths), grid (CTAs over all samples), vec2 (channel pairs stored as one word),
 * tma_epilogue (the output is staged in shared memory and written by TMA stores, the residual prefetched by TMA; 0 with
 * CVVAE_TMA_EPILOGUE=0 in the environment).  Writes the first min(n, count) values and returns count (15), or a negative
 * error code.  Launches nothing. */
int cvvae_conv_tc_plan(const cvvae_conv_desc* d, int32_t* out, int32_t n);
const char* cvvae_last_error(void);
int cvvae_abi_version(void);
/* Number of kernel launches issued through this library by the calling process (all threads). */
int64_t cvvae_launch_count(void);
/* Descriptor self-test used by the GPU test-suite: runs a 128xNx64 product (two 64-row wgmma chains, N in {64, 128,
 * 256}) whose A operand starts `row_shift` 128-byte rows into a TMA-written SWIZZLE_128B slab of 320 rows, with the given
 * base_offset field and with consecutive 8-row groups `sbo_rows` (8..16) slab rows apart.  a_rows: [320][64], out: fp32
 * [128][N].
 * (Decides how shifted conv taps may address one staged slab.)  16-bit dtypes only. */
int cvvae_probe_umma_shift(const void* a_rows, const void* b_rows, float* out, int32_t n, int32_t row_shift,
                           int32_t base_offset_mode, int32_t sbo_rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CVVAE_B200_H_ */
