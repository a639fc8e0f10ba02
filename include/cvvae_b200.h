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
 *     (convolution outputs: residual stream, q / k / v, attention output) is full fp32.  The video_io entry points of the
 *     inference script and cvvae_conv3d_stacked are 16-bit only and reject CVVAE_F32; cvvae_video_train_input and
 *     cvvae_video_output_u8 take all three.
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
  CVVAE_CONV_X_SHARED = 16,    /* x.B == 1: the same left operand for every batch item of y                       */
  /* y = max(alpha * acc + bias, 0) (-0 stored as +0), in the register epilogue: the conv + ReLU pairs of VGG16's
   * features[0:30] that LPIPS runs (lvdm/modules/autoencoding/lpips/loss/lpips.py:99-138).  CVVAE_F32 on the tensor-core
   * path only; refused with CVVAE_E_ARG before any launch for 16-bit dtypes, by cvvae_conv3d_direct,
   * cvvae_conv3d_stacked and by cvvae_conv3d on a descriptor the tensor-core path does not take, and together with a
   * residual, x2 / w2, gn_stats, up_time 2 or any other flag but CVVAE_CONV_TF32_OUT.  cvvae_conv_tc_plan reports the
   * same plan with it. */
  CVVAE_CONV_RELU = 32,
  /* With CVVAE_CONV_RELU only (refused otherwise, in the same places): y is stored rounded to the nearest TF32 value, for
   * an output whose only consumers are tensor-core products (the VGG16 layers that are not LPIPS taps), which would
   * otherwise read it with the low 13 mantissa bits dropped.  Same plan. */
  CVVAE_CONV_TF32_OUT = 64
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
/* f16_to_u8 over a batch, in any activation dtype: [B,3,T,H,W] (CVVAE_F16, CVVAE_BF16 or CVVAE_F32) -> uint8 [B,T,H,W,3],
 * both contiguous on the device, every element ((clamp(x,-1,1) + 1.0) * 127.5).to(uint8) as PyTorch evaluates it in the
 * tensor's dtype: 16-bit types round every intermediate to the type, CVVAE_F32 makes two single fp32 roundings.  NaN
 * inputs give an unspecified byte (the cast is undefined in PyTorch too).  A null pointer, B or a size < 1, an element
 * count 3*B*T*H*W beyond int64 or an unknown dtype is CVVAE_E_ARG before any launch.  One kernel launch. */
int cvvae_video_output_u8(const void* in_bcthw, uint8_t* out_bthwc, int32_t B, int32_t T, int32_t H, int32_t W,
                          int32_t dtype, void* stream);
/* The script's `transforms.Resize(size=(height, width))` on the uint8 frames (cvvae_inference_video.py:15-17,28), on the GPU:
 * antialiased bilinear (triangle filter, support scaled by the down-scale factor, round half up), uint8 [T,H,W,3] ->
 * out_thwc uint8 [T,OH,OW,3] and/or out_cthw 16-bit [3,T,OH,OW] = resized.half() / 127.5 - 1.0 (either may be NULL).
 * fp32 arithmetic: within 1 LSB of torchvision's fixed-point uint8 path (differs on < 1 % of the pixels). */
int cvvae_video_resize_u8(const uint8_t* thwc, uint8_t* out_thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t OH,
                          int32_t OW, int32_t dtype, void* stream);
/* The training data path's pre-processing (lvdm/data/decoder.py:99-109, 275-279; lvdm/data/transform.py:14-59, 66-121):
 * `torch.tensor(frames).permute(0, 3, 1, 2).float()`, `CoverResize(size)` or `Resize(min(size))`, `CenterCrop(size)`,
 * `(frames / 255 - 0.5) * 2`, as one pass.  uint8 thwc [T,H,W,3] -> out_cthw [3,T,OH,OW] (contiguous, F16 / BF16 / F32):
 * out(c,t,oy,ox) = pixel (oy + top, ox + left) of the frame resized to RH x RW by torchvision's antialiased bilinear
 * resize of a float tensor (ATen's CPU windows and weights, width reduced first, fp32 arithmetic, no rounding to uint8),
 * then (v / 255 - 0.5) * 2 in fp32, rounded once to the output type.  The crop window must lie inside RH x RW, else
 * CVVAE_E_ARG.  One kernel launch. */
int cvvae_video_train_input(const uint8_t* thwc, void* out_cthw, int32_t T, int32_t H, int32_t W, int32_t RH, int32_t RW,
                            int32_t top, int32_t left, int32_t OH, int32_t OW, int32_t dtype, void* stream);

/* Reconstruction quality: per-frame squared error and SSIM of two uint8 videos a, b: [T,H,W,3], contiguous, on the device.
 * They are the two ends of the inference script: its resized uint8 input (cvvae_inference_video.py:28) and the uint8
 * frames it writes (:47-50).
 *   acc: int64 [T][2], overwritten:  acc[t][0] = sum over (h,w,c) of (a-b)^2, the whole frame (exact)
 *                                    acc[t][1] = sum over the valid (h,w,c) of llrint(ssim * 2^32)
 * SSIM (Wang et al. 2004): per colour channel, at every (y,x) with 5 <= y < H-5, 5 <= x < W-5 (no padding), under the window
 * w = g (x) g, g = the 11-tap Gaussian exp(-k^2 / (2 * 1.5^2)) normalised to sum 1: means mu_a, mu_b, variances and
 * covariance E[a^2] - mu_a^2, E[b^2] - mu_b^2, E[ab] - mu_a mu_b; C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2;
 *   ssim = (2 mu_a mu_b + C1)(2 s_ab + C2) / ((mu_a^2 + mu_b^2 + C1)(s_a^2 + s_b^2 + C2)).
 * Frame SSIM = acc[t][1] / 2^32 / (3 (H-10) (W-10)); PSNR = 10 log10(255^2 * 3 H W / acc[t][0]).  The moments are exact
 * integer sums along rows and fp64 along columns, the formula is fp32; identical frames give exactly 2^32 per position.
 * Integer accumulation: bit-reproducible and independent of how the frames are split over calls.
 * T >= 0 (T == 0 launches nothing), H, W >= 11 and 3*H*W < 2^31, else CVVAE_E_ARG.  One kernel launch. */
int cvvae_frame_metrics(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, int64_t* acc,
                        void* stream);
/* cvvae_frame_metrics that also writes the SSIM map: map fp32 [T][H-10][3(W-10)], 4-byte aligned, overwritten with
 * map[t][y][3x + c] = the ssim above of channel c at pixel (y+5, x+5), the exact fp32 value whose llrint(ssim * 2^32) the
 * SSIM sum adds, so that sum over the map of llrint(v * 2^32) == acc[t][1].  acc is computed exactly as by
 * cvvae_frame_metrics, bit for bit.  The refusals of cvvae_frame_metrics, plus a NULL or misaligned map (CVVAE_E_ARG,
 * before any launch).  One kernel launch. */
int cvvae_frame_ssim_map(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, int64_t* acc,
                         float* map, void* stream);
/* Multi-scale SSIM (Wang, Simoncelli and Bovik 2003) of the same two videos, as per-level sums; the caller combines them.
 * Level 0 is the frames; level j+1 is the 2x2 average pool of level j, an odd extent zero-padded in front (output i of an
 * axis of odd length covers inputs 2i-1 and 2i, input -1 being 0; the divisor stays 4).  At each level j = 0..4, per
 * colour channel c and over the positions whose 11x11 window lies inside the level-j image, with the SSIM conventions
 * above (data range 255 at every level):
 *   acc: int64 [T][5][3][2], overwritten:  acc[t][j][c][0] = sum of llrint(cs * 2^32),  cs = (2 s_ab + C2) / (s_a^2 + s_b^2 + C2)
 *                                          acc[t][j][c][1] = sum of llrint(ssim * 2^32)
 * The level-j image is ceil(H / 2^j) x ceil(W / 2^j).  MS-SSIM(c) = prod_{j<4} max(cs_j, 0)^w_j * max(ssim_4, 0)^w_4 with
 * the means cs_j, ssim_j over the positions and w = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333); the frame's score is the
 * mean over c.  Levels 1-4 are kept as exact integer sums (uint16) in `workspace`: device memory of at least
 * cvvae_ms_ssim_workspace_bytes(T, H, W) bytes, 16-byte aligned.  Identical frames give exactly 2^32 per position.
 * T >= 0 (T == 0 launches nothing), H, W >= 161 and 3*H*W < 2^31, else CVVAE_E_ARG.  Nine kernel launches: the five
 * levels' scores and four pooling steps. */
int cvvae_frame_ms_ssim(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, void* workspace,
                        int64_t* acc, void* stream);
/* Bytes of the workspace cvvae_frame_ms_ssim needs for T frames of H x W px (T >= 0, H, W >= 1; else CVVAE_E_ARG). */
int64_t cvvae_ms_ssim_workspace_bytes(int32_t T, int32_t H, int32_t W);

/* LPIPS (VGG16, lpips v0.1) of two uint8 videos a, b: [T,H,W,3], contiguous, on the device, per frame:
 * LPIPS.forward(input, target) of the reference in eval mode (lvdm/modules/autoencoding/lpips/loss/lpips.py:46-64), with the
 * inputs taken as frame / 127.5 - 1.  The caller runs:
 *   cvvae_lpips_input: out fp32 [2T,H,W,32] channels-last, 16-byte aligned; image i < T is frame i of a, image T+i frame i of
 *     b.  Channel (kh*3 + kw)*3 + c of position (h, w) is s(h+kh-1, w+kw-1, c), s = ((p / 127.5 - 1) - shift_c) / scale_c
 *     (ScalingLayer, lpips.py:67-78: shift = (-0.030, -0.088, -0.188), scale = (0.458, 0.448, 0.450)), every operation an
 *     fp32 rounding as PyTorch evaluates it, stored rounded to the nearest TF32; 0 outside the frame (conv2d zero-pads the
 *     scaled input) and in channels 27..31.  conv1_1 then runs as a 1 x 1 convolution over these 32 channels with its
 *     weights packed [1][64][32] in the same channel order.  T >= 0 (T == 0 launches nothing), H, W >= 1.  One launch.
 *   the thirteen 3 x 3 convolutions of vgg16.features[0:30] (lpips.py:99-138) through cvvae_conv3d with CVVAE_CONV_RELU, plus
 *     CVVAE_CONV_TF32_OUT on the eight whose output only feeds the next convolution (all but the taps).
 *   cvvae_lpips_tap on each of the five taps relu1_2 .. relu5_3: f fp32 [2T,H,W,C] (C = 64, 128, 192, 256, 384 or 512),
 *     lin_w fp32 [C] (the 1x1 head lin{k}, no bias), acc int64 [T] overwritten with, per frame t,
 *       acc[t] = 2^32 * sum over the positions of sum_c w[c] (fa_c / n_a - fb_c / n_b)^2,
 *       n = sqrt(sum_c f_c^2 + 1e-10) + 1e-10   (normalize_tensor, lpips.py:141-143),
 *     with fa = image t, fb = image T+t.  The normalisation and the difference are fp64; each CTA's fp64 sum over its
 *     positions is rounded once to units of 2^-32 and added with an integer atomic: bit-reproducible, independent of the
 *     other frames in the call, exactly 0 for identical frames and the same bits with a and b swapped.  Range: H*W <= 2^23
 *     is checked (CVVAE_E_ARG); the heads must satisfy |w[c]| <= 32 (the Python loader refuses others; the entry point
 *     cannot read device memory before it launches) and the features must be finite.  Then |acc[t]| < 2^62.
 *     pooled: NULL, or fp32 [2T,H/2,W/2,C] that receives the 2 x 2 max pool (stride 2, floor) of all 2T images, the input
 *     of the next block, from the same pass, stored rounded to the nearest TF32 value (its only consumer is a
 *     convolution).  f, lin_w and pooled 16-byte aligned; T >= 0 (T == 0 launches nothing).
 *     One launch (plus a memset of acc).
 *   d_k(t) = acc[t] / 2^32 / (H_k W_k) and LPIPS(t) = sum_k d_k(t) are formed by the caller in fp64.  One group of frames
 *   costs 1 + 13 + 5 kernel launches. */
int cvvae_lpips_input(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, float* out, void* stream);
int cvvae_lpips_tap(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w, int64_t* acc,
                    float* pooled, void* stream);
/* LPIPS on AlexNet features (lpips v0.1 net='alex', the lpips package's default; torchvision alexnet().features[0:12]):
 * the same scaling, normalisation, heads and fixed-point sums as above, on five taps relu1 .. relu5 of C = 64, 192, 384,
 * 256, 256.  The caller runs, for T frame pairs of H x W px (H, W >= 31 for relu5 to have a position):
 *   cvvae_lpips_alex_input: conv1's input (11 x 11, stride 4, zero padding 2) with its 363 taps packed into channels:
 *     out fp32 [2T,h1,w1,384], h1 = (H-7)/4 + 1, w1 = (W-7)/4 + 1, 16-byte aligned, images as cvvae_lpips_input.  Channel
 *     (c*11 + kh)*11 + kw of position (oh, ow) is s(4 oh + kh - 2, 4 ow + kw - 2, c) with s exactly as cvvae_lpips_input
 *     computes it (TF32-rounded), 0 outside the frame and in channels 363..383: the order of the weight [64,3,11,11]
 *     flattened, so conv1 runs as a 1 x 1 convolution over 384 channels.  T >= 0 (T == 0 launches nothing), H, W >= 7.
 *     One launch.
 *   conv1 (cvvae_conv3d, CVVAE_CONV_RELU) -> relu1 [2T,h1,w1,64], fp32; cvvae_lpips_tap on it without a pool.
 *   cvvae_lpips_max_pool3s2: the 3 x 3 stride-2 max pool (floor, no padding) of features[2] and [5]: f fp32 [N,H,W,C] ->
 *     out fp32 [N,(H-3)/2+1,(W-3)/2+1,C], stored rounded to the nearest TF32 value (its only consumer is a convolution).
 *     N >= 0, H, W >= 3, C % 4 == 0, H*W*C < 2^31, both 16-byte aligned.  One launch.
 *   cvvae_lpips_pack5x5: conv2's 5 x 5 taps (zero padding 2) packed into channels: x fp32 [N,H,W,C] -> out fp32
 *     [N,H,W,25C], channel (kh*5 + kw)*C + c of (h, w) is x(h+kh-2, w+kw-2, c), 0 outside the image, an exact copy; conv2
 *     then runs as a 1 x 1 convolution over 25 * 64 = 1600 channels with its weights packed in that order.  N >= 0,
 *     H, W >= 1, C % 4 == 0, 25*H*W*C < 2^31, both 16-byte aligned.  One launch.
 *   conv2 -> relu2 [.., 192] and its tap; the pool; conv3 (3 x 3) -> relu3 [.., 384]; conv4 -> relu4 [.., 256];
 *     conv5 -> relu5 [.., 256].
 *   cvvae_lpips_tap_copy on relu3 and relu4: cvvae_lpips_tap (C = 256 or 384, no pool) that also writes `copy` fp32
 *     [2T,H,W,C], every value of f rounded to the nearest TF32, from the same pass: the input of the next convolution,
 *     while the tap itself stays fp32.  `copy` must not be NULL.  One launch (plus a memset of acc).
 *   cvvae_lpips_tap on relu5.  One group of frames costs 14 kernel launches.
 * Every index in these kernels is 64-bit across images and 32-bit within one (checked above). */
int cvvae_lpips_alex_input(const uint8_t* a_thwc, const uint8_t* b_thwc, int32_t T, int32_t H, int32_t W, float* out,
                           void* stream);
int cvvae_lpips_max_pool3s2(const float* f, int32_t N, int32_t H, int32_t W, int32_t C, float* out, void* stream);
int cvvae_lpips_pack5x5(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, float* out, void* stream);
int cvvae_lpips_tap_copy(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w, int64_t* acc,
                         float* copy, void* stream);
/* LPIPS maps (lpips spatial=True) for either network:
 *   cvvae_lpips_tap_map: cvvae_lpips_tap with `pooled` (VGG16's taps 1-4) or cvvae_lpips_tap_copy with `copy` (AlexNet's
 *     relu3, relu4), at most one of them set, else CVVAE_E_ARG; the same checks, the same acc bit for bit, the same side
 *     output.  It also writes map fp64 [T,H,W], 8-byte aligned (NULL or misaligned: CVVAE_E_ARG):
 *       map[t][h][w] = sum_c w[c] (fa_c / n_a - fb_c / n_b)^2 at that position, its own fp64 sum (not the fixed-point one),
 *     so that the mean of map[t] is d_k(t) up to the rounding of acc.  One launch (plus a memset of acc).
 *   cvvae_lpips_upsample_sum: taps fp64, the five tap maps [T,h_k,w_k] back to back (tap k from element
 *     sum_{j<k} T h_j w_j), tap_hw host int32 [10] = h_0, w_0, .., h_4, w_4 -> out fp32 [T,H,W] = sum over k of tap map k
 *     upsampled to H x W as nn.Upsample(size=(H, W), mode='bilinear', align_corners=False) does for fp32 tensors: per axis
 *     scale = (float)in / out, src = max(scale (dst + 0.5) - 0.5, 0) in fp32, i0 = (int)src, i1 = i0 + (i0 < in - 1),
 *     lambda = src - i0; the interpolation and the sum over k are fp64, rounded to fp32 once.  taps 8-byte and out 4-byte
 *     aligned; T >= 0 (T == 0 launches nothing), 1 <= H*W < 2^31, 1 <= h_k*w_k < 2^31, else CVVAE_E_ARG.  One launch.
 *   A group of frames then costs one launch more than its scores alone.  The map's mean over H x W is not exactly
 *   sum_k d_k: bilinear upsampling with the edges clamped does not preserve the mean (lpips behaves the same way). */
int cvvae_lpips_tap_map(const float* f, int32_t T, int32_t H, int32_t W, int32_t C, const float* lin_w, int64_t* acc,
                        float* pooled, float* copy, double* map, void* stream);
int cvvae_lpips_upsample_sum(const double* taps, int32_t T, int32_t H, int32_t W, const int32_t* tap_hw, float* out,
                             void* stream);

/* FVD's network: the Kinetics-400 I3D (InceptionI3d of the common PyTorch port) in fp32 with TF32 products, on N clips.
 * TF "SAME" padding per axis of extent n, kernel k, stride s: pad = max(k - s, 0) if n % s == 0 else max(k - n % s, 0),
 * front = pad / 2; the output extent is ceil(n / s).  The caller runs:
 *   cvvae_i3d_stem_input: x fp32 [N,3,T,H,W] contiguous (frames_to_training_input's output, 4-byte aligned) -> out fp32
 *     [N,TP,OH,OW,448] channels-last, 16-byte aligned, TP = ceil(T/2) + 2, OH = ceil(H/2), OW = ceil(W/2).  Channel
 *     ((j*7 + kh)*7 + kw)*3 + c of (u, oh, ow) is x(c, 2u - ft + j, 2oh - fh + kh, 2ow - fw + kw), j < 3, with ft, fh, fw the
 *     SAME front paddings of Conv3d_1a_7x7 (k = 7, s = 2), stored rounded to the nearest TF32 value; 0 outside the clip and
 *     in channels 441..447.  Conv3d_1a_7x7 then runs as a 3 x 1 x 1 stride-1 convolution (no offset) over these 448
 *     channels whose tap k holds the temporal taps 2k + j (tap 0: j = 0, 1, 2; taps 1 and 2: j = 1, 2; every other
 *     weight zero).  N >= 0 (N == 0 launches nothing), T, H, W >= 1, TP*OH*OW*112 < 2^31.  One launch.
 *   The 57 BN-folded convolutions (conv3d, BatchNorm3d(eps=1e-3) in eval mode, ReLU) through cvvae_conv3d with
 *     CVVAE_CONV_RELU and SAME offsets, plus CVVAE_CONV_TF32_OUT on all but Mixed_5c's branches (the head reads those).
 *   cvvae_i3d_max_pool3d: f fp32 [N,T,H,W,C] -> out fp32 [N,ceil(T/st),ceil(H/sh),ceil(W/sw),C], both channels-last,
 *     contiguous and 16-byte aligned, kernel / stride host int32 [3] (t, h, w), each 1..7: the maximum over the window with
 *     SAME zero padding (a tap outside the input counts as 0), an exact copy of the winning value.  N >= 0, T, H, W >= 1,
 *     C % 4 == 0, T*H*W*C < 2^31.  One launch.
 *   cvvae_i3d_head: f fp32 [N,T,7,7,C] (Mixed_5c, T >= 2), w fp32 [K][C] and bias fp32 [K] (the logits convolution) ->
 *     out fp64 [N,K] = bias + w . m, m[c] the mean over the T - 1 positions of AvgPool3d([2,7,7], stride 1) of channel c;
 *     all arithmetic fp64, bit-reproducible and independent of the other clips.  1 <= C <= 4096, K >= 1; out 8-byte
 *     aligned.  One launch.
 * Every refusal is CVVAE_E_ARG before any launch. */
int cvvae_i3d_stem_input(const float* x, int32_t N, int32_t T, int32_t H, int32_t W, float* out, void* stream);
int cvvae_i3d_max_pool3d(const float* f, int32_t N, int32_t T, int32_t H, int32_t W, int32_t C, const int32_t* kernel,
                         const int32_t* stride, float* out, void* stream);
int cvvae_i3d_head(const float* f, int32_t N, int32_t T, int32_t H, int32_t W, int32_t C, const float* w, const float* bias,
                   int32_t K, double* out, void* stream);

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
