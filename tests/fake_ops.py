"""Torch (CPU or CUDA) restatement of the operator set of ``cvvae_b200.ops.CudaOps``.

TEST DOUBLE ONLY - lives under tests/, is never importable from the product package.  Two uses:
  * CPU tests drive ``cvvae_b200.engine.Engine`` / the model wrapper through these operators to verify
    the graph wiring (padding modes, offsets, interleave, tiling, state-dict mapping) against the
    golden fixtures without a GPU;
  * GPU tests compare every CUDA kernel with the operator defined here on the same inputs
    (this file is the written-down semantics of each C-ABI entry point).
All maths in fp32 (or the input dtype when ``exact_dtype``), library calls only.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

PAD_ZERO, PAD_REPLICATE = 0, 1
GN_SUM_SCALE, GN_SQ_SCALE = 2.0 ** 20, 2.0 ** 18  # fixed-point statistics format of the C ABI


def _ncdhw(x):  # logical [B,T,H,W,C] -> [B,C,T,H,W]
    return x.permute(0, 4, 1, 2, 3)


class FakeOps:
    name = "fake"

    def __init__(self, compute_dtype=torch.float32):
        self.cd = compute_dtype
        self.launches = 0

    # ---- memory
    @staticmethod
    def empty(shape, dtype, device):
        return torch.full(tuple(shape), float("nan"), dtype=dtype, device=device)

    def empty_padded(self, B, T, H, W, Cc, dtype, device):
        p = torch.full((B, T, H + 2, W + 2, Cc), float("nan"), dtype=dtype, device=device)
        return p, p[:, :, 1:-1, 1:-1, :]

    # ---- conv
    def pack_weight(self, w):
        co, ci = w.shape[0], w.shape[1]
        return w.reshape(co, ci, -1).permute(2, 0, 1).contiguous()

    def conv(self, x, w, bias, *, kernel=(1, 1, 1), stride=(1, 1, 1), offset=(0, 0, 0), pad_t=PAD_ZERO, pad_hw=PAD_ZERO,
             up_time=1, residual=None, alpha=1.0, out=None, out_f32=False, bias_along_m=False, w_ld=0, cout=None,
             force=None, ref_taps=None, gn_stats=None, gn_groups=32, w_per_batch=False, x_shared=False, k_alg=None,
             sc_x=None, sc_w=None):
        self.launches += 1
        assert out is not None
        if w_per_batch or x_shared:
            # batched GEMM: one (x_b, w_b) product per batch item of `out`; a row bias is shared by the items
            for bi in range(out.shape[0]):
                self.conv(x[0:1] if x_shared else x[bi:bi + 1], w[bi:bi + 1] if w_per_batch else w, bias, kernel=kernel,
                          alpha=alpha, out=out[bi:bi + 1], out_f32=out_f32, bias_along_m=bias_along_m, w_ld=w_ld, cout=cout)
            self.launches -= out.shape[0]
            return out
        kt, kh, kw = kernel
        B, T, H, W, Ci = x.shape
        Co = cout if cout is not None else w.shape[1]
        wt = w[:, :Co, :Ci].to(self.cd)  # [taps, Co, Ci]
        wt = wt.permute(1, 2, 0).reshape(Co, Ci, kt, kh, kw)
        To = (out.shape[1] + 1) // 2 if up_time == 2 else out.shape[1]
        Ho, Wo = out.shape[2], out.shape[3]
        xin = _ncdhw(x).to(self.cd)

        def pads(n, no, k, s, off):
            lo = -off
            hi = (no - 1) * s + k - n - lo
            return lo, hi

        (tl, th) = pads(T, To, kt, stride[0], offset[0])
        (hl, hh) = pads(H, Ho, kh, stride[1], offset[1])
        (wl, wh) = pads(W, Wo, kw, stride[2], offset[2])

        def crop_neg(t, dim, lo, hi):
            # negative padding = the taps never reach that part of the input
            if lo < 0:
                t = t.narrow(dim, -lo, t.shape[dim] + lo)
                lo = 0
            if hi < 0:
                t = t.narrow(dim, 0, t.shape[dim] + hi)
                hi = 0
            return t, lo, hi

        xin, tl, th = crop_neg(xin, 2, tl, th)
        xin, hl, hh = crop_neg(xin, 3, hl, hh)
        xin, wl, wh = crop_neg(xin, 4, wl, wh)
        if hl or hh or wl or wh:
            xin = F.pad(xin, (wl, wh, hl, hh, 0, 0), mode="replicate" if pad_hw == PAD_REPLICATE else "constant")
        if tl or th:
            xin = F.pad(xin, (0, 0, 0, 0, tl, th), mode="replicate" if pad_t == PAD_REPLICATE else "constant")
        y = F.conv3d(xin, wt, None, stride=stride) * alpha
        assert y.shape[2:] == (To, Ho, Wo), (y.shape, (To, Ho, Wo))
        if bias is not None:
            if bias_along_m:
                y = y + bias.to(self.cd).reshape(B, 1, To, Ho, Wo)
            else:
                y = y + bias.to(self.cd).view(1, -1, 1, 1, 1)
        if up_time == 2:
            c = Co // 2
            y = y.reshape(B, 2, c, To, Ho, Wo).permute(0, 2, 3, 1, 4, 5).reshape(B, c, 2 * To, Ho, Wo)[:, :, 1:]
        y = y.permute(0, 2, 3, 4, 1)  # logical [B,T,H,W,C]
        if sc_w is not None:   # fused 1x1 shortcut: + sc_x @ sc_w^T, same accumulator (one rounding at the end)
            y = y + torch.einsum("bthwc,oc->bthwo", sc_x.to(self.cd), sc_w.to(self.cd))
        if residual is not None:
            y = y + residual.to(self.cd)
        out.copy_(y.to(out.dtype))
        if gn_stats is not None:  # sums of the STORED values per (sample, group)
            v = out.to(torch.float64)
            Bc, Tc, Hc, Wc, Cc = v.shape
            g = v.reshape(Bc, Tc * Hc * Wc, gn_groups, Cc // gn_groups)
            gn_stats[:, :, 0] += torch.round(g.sum(dim=(1, 3)) * GN_SUM_SCALE).to(torch.int64)
            gn_stats[:, :, 1] += torch.round((g * g).sum(dim=(1, 3)) * GN_SQ_SCALE).to(torch.int64)
        return out

    def conv_stacked(self, x, w_stk, bias, *, kt, cout, offset=(0, -1, -1), pad_t=PAD_ZERO, pad_hw=PAD_ZERO, out=None):
        # [KT][80][Cin] (row (kh*3+kw)*8 + c) -> packed [KT*9][Cout][Cin]
        ci = w_stk.shape[2]
        w = w_stk[:, :72].reshape(kt, 9, 8, ci)[:, :, :cout].reshape(kt * 9, cout, ci)
        return self.conv(x, w, bias, kernel=(kt, 3, 3), offset=offset, pad_t=pad_t, pad_hw=pad_hw, out=out)

    def new_stats(self, B, groups, device):
        return torch.zeros((B, groups, 2), dtype=torch.int64, device=device)

    # ---- norms
    def groupnorm(self, x, gamma, beta, groups, eps, *, per_frame=False, silu=True, out=None, stats=None):
        self.launches += 2
        B, T, H, W, Cc = x.shape
        xin = _ncdhw(x).to(self.cd)
        if per_frame:
            xin = xin.permute(0, 2, 1, 3, 4).reshape(B * T, Cc, H, W)
        if stats is not None:
            # statistics handed over by the producing conv: normalise with exactly those sums
            cnt = T * H * W * (Cc // groups)
            mean = (stats[:, :, 0].double() / GN_SUM_SCALE / cnt)
            var = (stats[:, :, 1].double() / GN_SQ_SCALE / cnt - mean * mean).clamp_min(0)
            rstd = (var + eps).rsqrt()
            mean_c = mean.repeat_interleave(Cc // groups, dim=1).to(self.cd).view(B, Cc, 1, 1, 1)
            rstd_c = rstd.repeat_interleave(Cc // groups, dim=1).to(self.cd).view(B, Cc, 1, 1, 1)
            y = (xin - mean_c) * rstd_c * gamma.to(self.cd).view(1, -1, 1, 1, 1) + beta.to(self.cd).view(1, -1, 1, 1, 1)
        else:
            y = F.group_norm(xin, groups, gamma.to(self.cd), beta.to(self.cd), eps)
        if silu:
            y = y * torch.sigmoid(y)
        if per_frame:
            y = y.reshape(B, T, Cc, H, W).permute(0, 1, 3, 4, 2)
        else:
            y = y.permute(0, 2, 3, 4, 1)
        if out is None:
            out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        out.copy_(y.to(out.dtype))
        return out

    def layernorm(self, x, gamma, beta, eps):
        self.launches += 1
        y = F.layer_norm(x.to(self.cd), (x.shape[-1],), gamma.to(self.cd), beta.to(self.cd), eps)
        return y.to(x.dtype)

    # ---- attention helpers
    def softmax_rows(self, s, cols, out):
        self.launches += 1
        out[:, :cols] = torch.softmax(s[:, :cols].float(), dim=-1).to(out.dtype)
        return out

    def attn_temporal(self, q, k, v):
        self.launches += 1
        B, T, H, W, Cc = q.shape
        qq, kk, vv = (t.to(self.cd).permute(0, 2, 3, 1, 4).reshape(B * H * W, T, Cc) for t in (q, k, v))
        s = torch.softmax(qq @ kk.transpose(1, 2) * (Cc ** -0.5), dim=-1)
        o = (s @ vv).reshape(B, H, W, T, Cc).permute(0, 3, 1, 2, 4)
        return o.to(q.dtype).contiguous()

    # ---- data movement
    def replicate_border(self, xpad):
        self.launches += 1
        H, W = xpad.shape[2], xpad.shape[3]
        xpad[:, :, 0, 1:W - 1] = xpad[:, :, 1, 1:W - 1]
        xpad[:, :, H - 1, 1:W - 1] = xpad[:, :, H - 2, 1:W - 1]
        xpad[:, :, :, 0] = xpad[:, :, :, 1]
        xpad[:, :, :, W - 1] = xpad[:, :, :, W - 2]

    def copy(self, x, out):
        self.launches += 1
        c = x.shape[-1]
        out[..., :c] = x
        if out.shape[-1] > c:
            out[..., c:] = 0
        return out

    def pack_taps_hw(self, x, out, kh, kw, offset=(0, 0), pad_hw=PAD_ZERO):
        self.launches += 1
        B, T, H, W, Cx = x.shape
        Ho, Wo = out.shape[2], out.shape[3]
        lo_h, lo_w = -offset[0], -offset[1]
        hi_h, hi_w = Ho + kh - 1 - H - lo_h, Wo + kw - 1 - W - lo_w
        xin = _ncdhw(x)
        xin = F.pad(xin.to(torch.promote_types(x.dtype, torch.float32)), (lo_w, hi_w, lo_h, hi_h, 0, 0),
                    mode="replicate" if pad_hw == PAD_REPLICATE else "constant").to(x.dtype)
        out.zero_()
        for a in range(kh):
            for b in range(kw):
                out[..., (a * kw + b) * Cx:(a * kw + b + 1) * Cx] = xin[:, :, :, a:a + Ho, b:b + Wo].permute(0, 2, 3, 4, 1)
        return out

    def blend(self, a, b, overlap, axis):
        self.launches += 1
        ov = overlap
        if axis == 0:
            wgt = (torch.arange(ov) / ov).view(1, 1, 1, -1, 1).to(b.device)  # CPU division, as the reference
            b[:, :, :, :ov] = ((1 - wgt) * a[:, :, :, -ov:] + wgt * b[:, :, :, :ov]).to(b.dtype)
        else:
            wgt = (torch.arange(ov) / ov).view(1, 1, -1, 1, 1).to(b.device)
            b[:, :, :ov] = ((1 - wgt) * a[:, :, -ov:] + wgt * b[:, :, :ov]).to(b.dtype)
        return b

    def launch_count(self):
        return self.launches
