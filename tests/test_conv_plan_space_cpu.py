"""The pure helpers of tests/test_gpu_conv_plan_space.py, which decide what that GPU test covers: slab counts per tile,
the TMA epilogue's ring wrap, the extent domain per level, and the choice of one case per signature (against a stub
planner)."""
import test_gpu_conv_plan_space as PS
from fake_ops import PAD_REPLICATE, PAD_ZERO


def _kind(**kw):
    k = {"view": "dense", "Cin": 128, "Cout": 128, "kernel": (3, 3, 3), "stride": (1, 1, 1), "offset": (-1, -1, -1),
         "pad_t": PAD_ZERO, "up_time": 1, "residual": False, "C2": 0, "gn": 32, "bias": True}
    k.update(kw)
    return k


def _plan(**kw):
    p = {"eligible": 1, "N_cta": 128, "NACC": 2, "TW": 64, "ROWS": 2, "TH": 4, "flat": 0, "NA": 3, "NB": 5,
         "tma_epilogue": 1, "tiles_w": 1, "tiles_h": 1}
    p.update(kw)
    return p


def test_slabs_per_tile():
    # stride 1: one slab per frame tap, column tap and channel block feeds all three row taps
    zero = _kind()
    # zero time padding (1, 1): the clip's first and last frames skip one frame tap
    assert [PS.slabs_per_tile(zero, t, 5) for t in range(5)] == [2 * 3 * 2, 9 * 2, 9 * 2, 9 * 2, 2 * 3 * 2]
    assert PS.slabs_per_tile(zero, 0, 1) == 3 * 2                        # one frame: both outer taps skipped
    causal = _kind(offset=(-2, -1, -1), pad_t=PAD_REPLICATE)
    assert {PS.slabs_per_tile(causal, t, 5) for t in range(5)} == {18}   # replicate: every tap loads
    assert PS.slabs_per_tile(_kind(C2=128), 2, 5) == 20                  # fused shortcut: one slab per block
    assert PS.slabs_per_tile(_kind(C2=64), 2, 5) == 19
    assert PS.slabs_per_tile(_kind(kernel=(1, 3, 3), offset=(0, -1, -1)), 0, 1) == 3 * 2
    # stride 2 in H: one row group per row tap (KHs = 1); stride 2 in time reads frames 2t - 2 .. 2t
    down = _kind(stride=(2, 2, 2), offset=(-2, 0, 0), pad_t=PAD_ZERO)
    assert [PS.slabs_per_tile(down, t, 5) for t in range(3)] == [9 * 2, 27 * 2, 27 * 2]
    assert PS.slabs_per_tile(_kind(Cin=32, kernel=(3, 1, 1), offset=(-2, 0, 0)), 0, 3) == 1   # hwpack: Cin 32, 1 block
    assert PS.slabs_per_tile(_kind(Cin=32, kernel=(1, 1, 1), offset=(0, 0, 0)), 0, 1, cb=32) == 1


def test_epilogue_wrap():
    k = _kind()
    p = _plan(NA=3)
    assert not PS.epilogue_wraps(k, p, 1, 0, 54)     # slot 0, then 1
    assert not PS.epilogue_wraps(k, p, 1, 0, 55)     # 1, 2
    assert PS.epilogue_wraps(k, p, 1, 0, 56)         # 2, then 3 -> slot 0 with the flipped parity
    assert PS.epilogue_wraps(k, _plan(NA=2), 1, 0, 55) and not PS.epilogue_wraps(k, _plan(NA=2), 1, 0, 54)
    # a block past Cout is not staged: Cout = 64 in a 128-channel CTA never wraps at slot 2
    assert not PS.epilogue_wraps(_kind(Cout=64), p, 1, 0, 56)
    # up_time = 2 drops the first channel half at t = 0: only block 1 is staged (slot 2 + 1 wraps, slot 0 + 1 not)
    up = _kind(Cout=128, up_time=2)
    assert PS.epilogue_wraps(up, p, 0, 0, 56) and not PS.epilogue_wraps(up, p, 0, 0, 54)
    up256 = _kind(Cout=512, up_time=2)
    p256 = _plan(N_cta=256, NA=4)
    assert not PS.epilogue_wraps(up256, p256, 0, 0, 4 * 27)      # blocks 0-3 are the dropped half at t = 0
    assert PS.epilogue_wraps(up256, p256, 1, 0, 4 * 27 + 1)
    sigs = PS.tile_signatures(_kind(C2=128), _plan(NA=3), 5, 5)
    assert {s[-3:] for s in sigs} == {(3, 14 % 3, True), (3, 20 % 3, True)}      # 12 + 2 at the clip's ends
    assert {s[-1] for s in PS.tile_signatures(_kind(), _plan(tma_epilogue=0), 5, 5)} == {None}


def test_extent_domain_per_level():
    # the decoder: latent tiles 1-72, 2^l times that at level l
    assert sorted(PS.extent_domain("sd21", "dec", 0)) == list(range(1, 73))
    assert sorted(PS.extent_domain("sd3", "dec", 3)) == list(range(8, 577, 8))
    # the encoder: sd21 halves without padding, so tiles below 8 px are not encodable; sd3 pads (1, 1)
    assert PS.extent_domain("sd21", "enc", 0) == {n: n for n in range(8, 577)}
    assert sorted(PS.extent_domain("sd21", "enc", 3)) == list(range(1, 73))
    assert PS.extent_domain("sd21", "enc", 1)[4] == 8 and PS.extent_domain("sd21", "enc", 1)[288] == 576
    assert sorted(PS.extent_domain("sd3", "enc", 0)) == list(range(1, 577))
    assert sorted(PS.extent_domain("sd3", "enc", 3)) == list(range(1, 73))
    assert PS.extent_domain("sd3", "enc", 2)[1] == 1 and PS.extent_domain("sd3", "enc", 2)[2] == 5
    for lv in range(PS.LEVELS):   # every extent is reached from its smallest tile
        for ext, n in PS.extent_domain("sd3", "enc", lv).items():
            assert PS.level_extent("sd3", "enc", lv, n) == ext and PS.level_extent("sd3", "enc", lv, n - 1) != ext
    assert [PS.level_frames("enc", lv, 17) for lv in range(4)] == [17, 9, 9, 5]
    assert [PS.level_frames("dec", lv, 5) for lv in range(4)] == [5, 9, 9, 17]


def _stub_plan(kind, site, t_in, t_out, nh, nw):
    """A planner in the shape of conv_tc_plan: TW 16 below 64 px, else 32; NACC halves below 40 CTAs per sample;
    ineligible at 3 px."""
    _, _, _, yl, _ = site["where"]
    h, w = PS.level_extent("sd3", "dec", yl, nh), PS.level_extent("sd3", "dec", yl, nw)
    if w == 3:
        return None
    tw = 16 if w < 64 else 32
    rows = 128 // tw
    nacc = 2
    while True:
        th = rows * nacc
        tiles_w, tiles_h = -(-w // tw), -(-h // th)
        if nacc == 1 or t_out * tiles_w * tiles_h >= 40:
            break
        nacc //= 2
    return {"eligible": 1, "N_cta": 128, "NACC": nacc, "TW": tw, "ROWS": rows, "TH": th, "flat": 0, "NA": 4, "NB": 6,
            "tma_epilogue": 1, "tiles_w": tiles_w, "tiles_h": tiles_h}


def test_representative_selection_against_a_stub_planner():
    kind = _kind(offset=(-2, -1, -1), pad_t=PAD_REPLICATE)
    site = {"where": ("sd3", "dec", 0, 0, False), "frames": {(1, 1), (2, 2), (3, 3), (5, 5)}}
    kind["sites"] = [site]
    calls = []

    def plan_fn(*a):
        calls.append(a[2:])
        return _stub_plan(*a)
    best, queries = PS.select(kind, plan_fn)
    assert queries == len(calls)
    # W classes: 72 latent extents -> 9 classes of ceil(w / 8); frames 1..5 bisected, never all four per (h, class)
    assert len(calls) < 72 * 9 * 4
    assert {c[3] for c in calls} <= {1, 9, 17, 25, 33, 41, 49, 57, 65}
    sigs = {s[:8] for s in best}
    assert sigs == {(128, 1, 16, 8, 0, 4, 6, 1), (128, 2, 16, 8, 0, 4, 6, 1), (128, 1, 32, 4, 0, 4, 6, 1),
                    (128, 2, 32, 4, 0, 4, 6, 1)}
    for sig, (score, shape) in best.items():
        si, t_in, t_out, nh, nw = shape
        plan = _stub_plan(kind, site, t_in, t_out, nh, nw)
        assert plan is not None and sig in PS.tile_signatures(kind, plan, t_in, t_out)
        assert score == PS.case_score(kind, PS.tile_properties(plan, nh, nw), t_out, nh, nw)
        # no shape in the domain reaching the signature comes earlier: more of the properties, enough elements for
        # gate 3, fewer positions
        for t_i, t_o in site["frames"]:
            for h in range(1, 73):
                for w in range(1, 73):
                    p = _stub_plan(kind, site, t_i, t_o, h, w)
                    if p is None or sig not in PS.tile_signatures(kind, p, t_i, t_o):
                        continue
                    other = PS.case_score(kind, PS.tile_properties(p, h, w), t_o, h, w)
                    assert other >= score, (sig, shape, (t_o, h, w))
    # the 2-accumulator plans come with a partial, ragged and interior tile; NACC = 1 cannot have a partial one
    for sig, (score, _) in best.items():
        assert score[:2] == (-3 if sig[1] == 2 else -2, False), (sig, score)
    # 4096 elements at 128 channels: 32 positions
    assert PS.case_score(kind, (True,) * 3, 1, 4, 7)[1] and not PS.case_score(kind, (True,) * 3, 1, 4, 8)[1]
