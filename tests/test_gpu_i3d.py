"""FVD's I3D on the H100: the stem packing and the max pool bit for bit against torch, the head against fp64 under a
derived bound, the whole embedding against the fp64 restatement (tests/i3d_ref.py) gated by the error of PyTorch's own
TF32 evaluation, bit-identity across calls, groupings and batches, embed_clips against the network, launch counts, flat
memory and the refusals."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import i3d_ref as R

pytestmark = pytest.mark.gpu
_WORST = {}


def _bits(x):
    return x.contiguous().view(torch.int32)


def _lib():
    from cvvae_b200 import _lib as L
    return L, L.load()


@pytest.fixture(scope="module")
def net():
    from cvvae_b200 import I3D
    sd = R.make_state_dict(11)
    return sd, I3D.from_state_dict(sd)


def _clip(kind, T, H, W, seed):
    """uint8 [T, H, W, 3] on the device: noise, a smooth moving pattern, a flat colour or a moving vertical edge."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "noise":
        return torch.randint(0, 256, (T, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    t = torch.arange(T, device="cuda", dtype=torch.float64)[:, None, None, None]
    y = torch.arange(H, device="cuda", dtype=torch.float64)[None, :, None, None]
    x = torch.arange(W, device="cuda", dtype=torch.float64)[None, None, :, None]
    c = torch.arange(3, device="cuda", dtype=torch.float64)
    if kind == "smooth":
        v = 127.5 + 100 * torch.sin(x / 17 + t / 3 + c) * torch.cos(y / 23 - t / 5 + 2 * c)
    elif kind == "flat":
        v = torch.zeros((T, H, W, 3), device="cuda", dtype=torch.float64) + torch.tensor([40.0, 170.0, 230.0], device="cuda")
    else:
        v = torch.where(x < W / 4 + 7 * t, 230.0, 20.0) + 0 * y + 10 * c
    return v.round().clamp(0, 255).to(torch.uint8).expand(T, H, W, 3).contiguous()


def _prepared(clips):
    from cvvae_b200 import frames_to_training_input
    return torch.cat([frames_to_training_input(c, 224, "short", torch.float32) for c in clips])


def _stem_packed(x):
    """torch's packing of the prepared clips [N, 3, T, H, W]: [N, TP, ho, wo, 448], channel ((j*7 + kh)*7 + kw)*3 + c
    the frame 2u - ft + j, SAME-padded, TF32-rounded."""
    from cvvae_b200.fvd import same_padding
    N, _, T, H, W = x.shape
    (ft, _, to), (fh, _, ho), (fw, _, wo) = same_padding(T, 7, 2), same_padding(H, 7, 2), same_padding(W, 7, 2)
    TP = to + 2
    xp = F.pad(x, (fw, 7, fh, 7, ft, 2 * TP + 1 - T - ft))
    out = torch.zeros((N, TP, ho, wo, 448), device=x.device)
    for j in range(3):
        frames = xp[:, :, j:j + 2 * TP - 1:2]                                   # [N, 3, TP, Hp, Wp]: frames 2u + j
        patches = frames.unfold(3, 7, 2).unfold(4, 7, 2)[:, :, :, :ho, :wo]   # [N, 3, TP, ho, wo, 7, 7]
        out[..., j * 147:(j + 1) * 147] = patches.permute(0, 2, 3, 4, 5, 6, 1).reshape(N, TP, ho, wo, 147)
    return R.tf32(out)


@pytest.mark.parametrize("N,T,H,W", [(2, 9, 224, 224), (1, 16, 224, 224), (2, 17, 224, 224), (1, 10, 37, 45),
                                     (3, 11, 8, 9), (1, 1, 7, 7)])
def test_stem_packing_is_torch_bit_for_bit(N, T, H, W):
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(T * H + W)
    x = torch.randn((N, 3, T, H, W), generator=g, device="cuda")
    TP, ho, wo = (T + 1) // 2 + 2, (H + 1) // 2, (W + 1) // 2
    out = torch.full((N, TP, ho, wo, 448), float("nan"), device="cuda")
    L.check(lib.cvvae_i3d_stem_input(x.data_ptr(), N, T, H, W, out.data_ptr(), L._stream(x)), "stem input")
    want = _stem_packed(x)
    assert torch.equal(_bits(out), _bits(want))
    # the borders read padding: the first packed frame's j = 0 block at T = 16 (ft = 2), and channels 441.. are zero
    assert (out[..., 441:] == 0).all()
    if T == 16:
        assert (out[:, 0, :, :, :294] == 0).all() and (out[:, -1] == 0).all()


@pytest.mark.parametrize("T", [9, 16, 17])
def test_224_clips_pass_through_unresized(T):
    """A 224 x 224 clip's network input is (x / 255 - 0.5) * 2 in IEEE fp32 arithmetic, bit for bit.  (The quotient is
    formed in fp64 and rounded: x / 255 has a periodic binary expansion, so that is the correctly rounded fp32 quotient.
    PyTorch's CUDA division by a scalar multiplies by the reciprocal instead, which differs in the last bit.)"""
    clip = _clip("noise", T, 224, 224, T)
    clip.view(-1, 3)[:256] = torch.arange(256, device="cuda", dtype=torch.uint8)[:, None]   # every byte in every channel
    x = _prepared([clip])
    want = (((clip.double() / 255).float() - 0.5) * 2).permute(3, 0, 1, 2)[None]
    assert torch.equal(_bits(x), _bits(want))


_POOLS = [(2, 8, 112, 112, 64, (1, 3, 3), (1, 2, 2)), (1, 9, 56, 56, 192, (1, 3, 3), (1, 2, 2)),
          (2, 9, 28, 28, 480, (3, 3, 3), (2, 2, 2)), (1, 5, 14, 14, 832, (2, 2, 2), (2, 2, 2)),
          (3, 3, 7, 7, 832, (3, 3, 3), (1, 1, 1)), (2, 5, 13, 11, 16, (3, 3, 3), (2, 2, 2)),
          (1, 3, 9, 7, 8, (2, 2, 2), (2, 2, 2)), (2, 1, 15, 17, 4, (1, 3, 3), (1, 2, 2)), (1, 2, 3, 5, 12, (3, 3, 3), (1, 1, 1))]


@pytest.mark.parametrize("N,T,H,W,C,k,s", _POOLS)
def test_max_pool_is_torch_bit_for_bit(N, T, H, W, C, k, s):
    """F.pad (SAME, zeros) + F.max_pool3d on ReLU outputs, as the network pools them."""
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(C + H)
    f = R.tf32(torch.relu(torch.randn((N, T, H, W, C), generator=g, device="cuda")))
    o = [-(-n // st) for n, st in zip((T, H, W), s)]
    out = torch.full((N, *o, C), float("nan"), device="cuda")
    L.check(lib.cvvae_i3d_max_pool3d(f.data_ptr(), N, T, H, W, C, (ctypes.c_int32 * 3)(*k), (ctypes.c_int32 * 3)(*s),
                                     out.data_ptr(), L._stream(f)), "max pool")
    want = R.max_pool(f.permute(0, 4, 1, 2, 3), k, s).permute(0, 2, 3, 4, 1)
    assert torch.equal(_bits(out), _bits(want))


@pytest.mark.parametrize("N,T5,K", [(3, 2, 400), (2, 3, 400), (1, 5, 10)])
def test_head_against_fp64(N, T5, K):
    """The head in fp64 against the restatement's in fp64: the two differ only in the order of fp64 sums, so every entry
    is within (T5 * 49 + C + 8) * 2^-52 * (|b| + sum_c |w_c| max|f|) (both sides' summation bound, doubled)."""
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(T5 * K)
    f = 3 * torch.rand((N, T5, 7, 7, 1024), generator=g, device="cuda")
    w = torch.randn((K, 1024), generator=g, device="cuda") / 32
    b = torch.randn(K, generator=g, device="cuda")
    out = torch.full((N, K), float("nan"), device="cuda", dtype=torch.float64)
    L.check(lib.cvvae_i3d_head(f.data_ptr(), N, T5, 7, 7, 1024, w.data_ptr(), b.data_ptr(), K, out.data_ptr(),
                               L._stream(f)), "head")
    sd = {"logits.conv3d.weight": w.double()[:, :, None, None, None], "logits.conv3d.bias": b.double()}
    want = R.head(f.double().permute(0, 4, 1, 2, 3), sd)
    bound = (T5 * 49 + 1024 + 8) * 2.0 ** -52 * (b.double().abs() + w.double().abs().sum(1) * f.max().double())
    assert ((out - want).abs() <= bound).all(), ((out - want).abs() / bound).max().item()


_KINDS = ("noise", "smooth", "flat", "edge")


@pytest.mark.parametrize("T", [9, 16, 17])
def test_embedding_against_fp64(net, T):
    """max |ours - fp64| <= 3 max |torch_tf32 - fp64| + 1e-6 max |fp64| per clip: the gate of the LPIPS metrics.  torch_tf32
    is PyTorch's default fp32 evaluation of the restatement (cuDNN, TF32 on), the stem's operands rounded to TF32."""
    sd, i3d = net
    clips = torch.stack([_clip(kind, T, 224, 224, 100 + T) for kind in _KINDS])
    ours = i3d(clips)
    x = _prepared(clips)
    fp64 = R.embed(x, sd).cpu()
    tf32 = R.embed(x, sd, tf32=True).double().cpu()
    assert ours.dtype == torch.float64 and ours.shape == (4, 400)
    for i, kind in enumerate(_KINDS):
        err, ref_err = (ours[i] - fp64[i]).abs().max().item(), (tf32[i] - fp64[i]).abs().max().item()
        gate = 3 * ref_err + 1e-6 * fp64[i].abs().max().item()
        _WORST[(T, kind)] = err / gate
        print(f"T={T} {kind}: ours {err:.3e}, torch TF32 {ref_err:.3e}, ratio to gate {err / gate:.3f}, "
              f"ours / torch {err / max(ref_err, 1e-300):.2f}")
        assert err <= gate, (T, kind, err, ref_err)


def test_embedding_is_bit_identical_across_calls_groups_and_batches(net):
    _, i3d = net
    clips = torch.stack([_clip(kind, 9, 224, 224, 7) for kind in _KINDS])
    first = i3d(clips)
    assert torch.equal(first, i3d(clips))
    i3d._group_bytes, saved = 1, i3d._group_bytes   # one clip per group
    try:
        assert i3d.group(9) == 1
        assert torch.equal(first, i3d(clips))
    finally:
        i3d._group_bytes = saved
    assert torch.equal(first[2:3], i3d(clips[2:3]))
    assert torch.equal(first[1:3], i3d(clips[1:3].flip(0)).flip(0))


def test_embed_clips_equals_the_network(net):
    """Mixed lengths and source sizes, host (numpy and tensor) and device items, batches of 2 keyed on (T, H, W)."""
    from cvvae_b200 import embed_clips
    _, i3d = net
    specs = [(9, 224, 224, "noise"), (9, 224, 224, "smooth"), (9, 224, 224, "edge"), (16, 240, 320, "smooth"),
             (16, 240, 320, "noise"), (17, 96, 128, "edge"), (9, 224, 224, "flat"), (12, 300, 200, "noise")]
    items, want = [], []
    for n, (T, H, W, kind) in enumerate(specs):
        clip = _clip(kind, T, H, W, n)
        want.append(i3d(clip[None])[0])
        items.append(clip.cpu().numpy() if n % 3 == 0 else clip.cpu() if n % 3 == 1 else clip)
    got = list(embed_clips(i3d, items, batch_size=2))
    assert len(got) == len(specs)
    for n, (g, w) in enumerate(zip(got, want)):
        assert g.device.type == "cpu" and g.dtype == torch.float64 and torch.equal(g, w), n


def test_launch_count(net):
    """N preparation launches, then i3d.launches per group of clips."""
    L, lib = _lib()
    _, i3d = net
    clips = torch.stack([_clip("noise", 9, 64, 80, n) for n in range(3)])
    i3d(clips)
    torch.cuda.synchronize()
    before = lib.cvvae_launch_count()
    i3d(clips)
    assert lib.cvvae_launch_count() - before == 3 + i3d.launches == 75
    from cvvae_b200.fvd import i3d_plan
    i3d._group_bytes, saved = 2 * i3d_plan(9).clip_bytes(), i3d._group_bytes   # two clips per group
    try:
        assert i3d.group(9) == 2
        before = lib.cvvae_launch_count()
        i3d(clips)
        assert lib.cvvae_launch_count() - before == 3 + 2 * i3d.launches
    finally:
        i3d._group_bytes = saved


def test_embed_clips_memory_is_flat_in_the_number_of_clips(net):
    from cvvae_b200 import embed_clips
    _, i3d = net
    clip = _clip("smooth", 9, 120, 160, 3).cpu()

    def peak(n):
        list(embed_clips(i3d, [clip] * 2, batch_size=2))   # warm: the pinned staging and the allocator's pools
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = list(embed_clips(i3d, [clip] * n, batch_size=2))
        torch.cuda.synchronize()
        assert len(out) == n
        return torch.cuda.max_memory_allocated() - base

    small, large = peak(4), peak(12)
    assert large <= small + (1 << 20), (small, large)


def test_refusals_before_any_launch(net):
    from cvvae_b200 import embed_clips
    L, lib = _lib()
    _, i3d = net
    good = _clip("noise", 9, 32, 32, 0)
    before = lib.cvvae_launch_count()
    for bad, msg in ((good[None].float(), "CUDA uint8"), (good[None].cpu(), "CUDA uint8"), (good, "CUDA uint8"),
                     (good[None, :8], "at least 9 frames"), (good[None, ..., :2], "CUDA uint8")):
        with pytest.raises(ValueError, match=msg):
            i3d(bad)
    for bad, msg in ((good[:8], "T >= 9"), (good.float(), "uint8"), (np.zeros((9, 8, 8, 3), np.int16), "uint8")):
        with pytest.raises(ValueError, match=msg):
            list(embed_clips(i3d, [bad]))
    assert lib.cvvae_launch_count() == before


def test_report_worst_ratio():
    if _WORST:
        (T, kind), r = max(_WORST.items(), key=lambda kv: kv[1])
        print(f"largest ratio of our error to the gate: {r:.3f} (T={T}, {kind})")
