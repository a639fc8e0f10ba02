"""conv_tc at every tile plan its planner chooses for the network's layers at any input size, fp16, bf16 and fp32,
against fp64.

The planner (conv_tc_plan in cvvae_b200/csrc/conv_tc.cu) picks N_cta, NACC, the tile TW x ROWS and the ring depths
NA / NB from the output extents, so the size of a user's video decides which kernel code runs.  The tiler's last tile
in a row or column is anywhere from 1 to 576 px (stride 448), and clips below 577 px are not tiled, so every extent
occurs.  This file
  1. records the layer kinds of the network: the conv calls of small real-width encode and decode passes, sd21 and sd3,
     at every frame count the codec produces for 1-17 input frames (17 is also the streaming chunk), everything but the
     extents kept (record_kinds).  The attention GEMMs (batched, fp32 logits) are tests/test_gpu_attention16.py's;
  2. enumerates, per kind, the plan of every output extent the kind sees from pixel tiles of 1-576 px (latent tiles
     of 1-72), through cvvae_conv_tc_plan on descriptors with aligned dummy pointers (the planner reads pointer values
     for alignment and never dereferences them).  Skipped without loss, because no ceiling of the planner changes:
       - W within one ceil(W / 8) class: every W-dependent quantity is ceil(W / TW) with TW a multiple of 8 (flat
         problems: the positions P within one ceil(P / 128) class, ceil(P / (NACC * 128)));
       - the frame counts strictly between two with equal plans: T_out enters only as a factor of the CTA count that
         stops the NACC halving, so NACC is monotone in T_out and the rest of the plan follows from NACC;
  3. splits every tile of a plan into a signature: the plan fields SIG_FIELDS, the K loop (KHs and the slab count mod
     NA, which zero-padded frame taps change at the clip's ends) and whether the TMA epilogue's staging slots wrap past
     NA (tile_signatures);
  4. picks per reachable (signature, kind) the smallest shape that reaches it, preferring shapes with a tile whose
     nacc_eff < NACC, a W-ragged tile and an interior tile (select; a case with few elements runs as a batch, the plan
     being per sample, so that gate 3 averages over enough of them), confirms its plan through CudaOps.conv_tc_plan on
     the real tensors, and runs it through network_audit.AuditOps(CudaOps()): fp64 at the sample frames, gates 1-3, the
     statistics gate, TF32 operand reading in fp32, NaN-filled outputs.  16-bit cases also run with the register
     epilogue (CVVAE_TMA_EPILOGUE=0) and into an output at an odd element offset (word stores off, so the general
     epilogue loop); all three must be bit-identical, statistics included;
  5. requires, for every NA of a TMA-epilogue plan, tiles whose staging wraps and tiles whose staging does not.  The
     network's 3x3x3 / 1x3x3 slab counts never wrap at NA = 3; SYNTHETIC adds API-admissible kinds for that.
The reachable set is frozen for 132-SM devices (H100 SXM) in tests/golden/conv_plan_space_132.json; NACC halving
depends on the SM count, so on another count the set is recorded and every reachable signature must still run and pass.
Rows go to conv_plan_space.json in test_gpu_ops.OUT.
"""
import ctypes as C
import json
import math
import os
import time

import pytest
import torch

import test_gpu_ops
from fake_ops import PAD_REPLICATE, PAD_ZERO

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT = test_gpu_ops.OUT

SIG_FIELDS = ("N_cta", "NACC", "TW", "ROWS", "flat", "NA", "NB", "tma_epilogue")
PIXEL_TILE, LATENT_TILE = 576, 72      # the model's default tile_spatial_size and its latent size
LEVELS = 4
ENC_FRAMES = tuple(range(1, 18))       # one chunk (en_de_n_frames_a_time 16, plus the shared first frame)
REC_PIXELS = 40                        # recording extent: 40 / 20 / 10 / 5, none of them 2 more than another
CB16 = 64                              # channels per operand block in 16-bit storage
GATE3_ELEMS = 4096


# ------------------------------------------------------------------------------------------ pure helpers
def level_extent(variant, direction, level, n):
    """Extent at `level` of a tile of extent n: encoder levels stride-2 3-tap convs, pads (0, 1) sd21 / (1, 1) sd3
    (Engine.encoded_hw); decoder level l is 2^l times the latent extent."""
    if direction == "dec":
        return n << level
    for _ in range(level):
        n = (n + (2 if variant == "sd3" else 1) - 3) // 2 + 1
    return n


def level_frames(direction, level, t):
    """Frames at `level` of a pass over t frames: the encoder halves them ((t - 1) // 2 + 1) into levels 1 and 3, the
    decoder's up-samplers into levels 1 and 3 double them less one (Engine.encoded_frames / decoded_frames)."""
    for lv in range(level):
        if lv % 2 == 0:
            t = (t - 1) // 2 + 1 if direction == "enc" else 2 * t - 1
    return t


def extent_domain(variant, direction, level):
    """{extent at `level`: the smallest tile extent giving it} over tiles of 1-576 px (encoder) / 1-72 latent (decoder)
    that the network can encode (sd21 halves without padding: a tile needs 8 px for a one-position latent)."""
    dom = {}
    for n in range(1, (PIXEL_TILE if direction == "enc" else LATENT_TILE) + 1):
        if level_extent(variant, direction, LEVELS - 1, n) >= 1:
            dom.setdefault(level_extent(variant, direction, level, n), n)
    return dom


def slabs_per_tile(kind, t, t_in, cb=CB16):
    """Activation slabs of the tile at output frame t: one per valid frame tap, row group, column tap and channel block
    (for_each_slab), then one per shortcut channel block."""
    kt_, kh, kw = kind["kernel"]
    kh_s = kh if kind["stride"][1] == 1 else 1
    taps = 0
    for j in range(kt_):
        ti = t * kind["stride"][0] + j + kind["offset"][0]
        if 0 <= ti < t_in or kind["pad_t"] == PAD_REPLICATE:
            taps += 1
    return taps * (kh // kh_s) * kw * -(-kind["Cin"] // cb) + -(-kind["C2"] // cb)


def epilogue_wraps(kind, plan, t, n0, slabs):
    """Whether the TMA epilogue stages a channel block of this tile in slot epi_slot + c >= NA (the parity flip), for
    the blocks it writes: inside Cout and, for up_time = 2, not the dropped first half at t = 0 (epi_block)."""
    epi = slabs % plan["NA"]
    co = kind["Cout"]
    for c in range(plan["N_cta"] // CB16):
        g = n0 + c * CB16
        if g >= co:
            continue
        if kind["up_time"] == 2 and 2 * t + g // (co // 2) - 1 < 0:
            continue
        if epi + c >= plan["NA"]:
            return True
    return False


def tile_signatures(kind, plan, t_in, t_out):
    """The signatures of the tiles of one frame count: plan fields, KHs, slab count mod NA, epilogue wrap (None
    without the TMA epilogue)."""
    base = tuple(plan[k] for k in SIG_FIELDS)
    kh_s = kind["kernel"][1] if kind["stride"][1] == 1 else 1
    out = set()
    for t in range(t_out):
        s = slabs_per_tile(kind, t, t_in)
        for n0 in range(0, kind["Cout"], plan["N_cta"]):
            wrap = epilogue_wraps(kind, plan, t, n0, s) if plan["tma_epilogue"] else None
            out.add(base + (kh_s, s % plan["NA"], wrap))
    return out


def tile_properties(plan, h, w):
    """(a tile with nacc_eff < NACC, a tile ragged in W, an interior tile) of output extents h x w (flat: w
    positions)."""
    if plan["flat"]:
        span = plan["NACC"] * 128
        last = w - (plan["tiles_w"] - 1) * span
        return -(-last // 128) < plan["NACC"], w % 128 != 0, w >= span
    last = h - (plan["tiles_h"] - 1) * plan["TH"]
    return -(-last // plan["ROWS"]) < plan["NACC"], w % plan["TW"] != 0, w >= plan["TW"] and h >= plan["TH"]


def site_shapes(kind, site):
    """The domain of one site of a kind, as query groups [(frames, (h, tile h), members)]: frames the (T_in, T_out)
    pairs in T_out order, members [(w, tile w)] the W extents of one ceil(W / 8) class.  Flat: frames [(1, 1)], h None,
    members [(P, (T_in, tile h, tile w))] the positions of one ceil(P / 128) class."""
    variant, direction, xl, yl, _ = site["where"]
    frames = sorted(site["frames"], key=lambda f: (f[1], f[0]))
    hs = extent_domain(variant, direction, yl)
    if kind["view"] == "flat":
        classes = {}
        for (t_in, _) in frames:
            for eh, nh in hs.items():
                for ew, nw in hs.items():
                    p = t_in * eh * ew
                    classes.setdefault(-(-p // 128), {}).setdefault(p, (t_in, nh, nw))
        return [([(1, 1)], None, sorted(members.items())) for _, members in sorted(classes.items())]
    classes = {}
    for ew, nw in sorted(hs.items()):
        classes.setdefault(-(-ew // 8), []).append((ew, nw))
    return [(frames, (eh, nh), cls) for eh, nh in sorted(hs.items()) for _, cls in sorted(classes.items())]


def select(kind, plan_fn):
    """Enumerate the kind's domain through plan_fn(kind, site, T_in, T_out, tile h, tile w) -> plan dict (None: not
    eligible) and pick, per reachable signature, the first shape in case_score order.
    Returns ({signature: (score, shape)}, plan queries); a shape is (site index, T_in, T_out, tile h, tile w)."""
    best, queries = {}, 0
    sig_cache = {}
    for si, site in enumerate(kind["sites"]):
        for frames, hn, members in site_shapes(kind, site):
            if hn is None:     # flat: one query per class of positions, at its smallest member
                t0, nh0, nw0 = members[0][1]
                plan = plan_fn(kind, site, t0, 1, nh0, nw0)
                queries += 1
                if plan is None:
                    continue
                sigs = tile_signatures(kind, plan, 1, 1)
                for p, (t_in, nh, nw) in members:
                    _offer(best, sigs, case_score(kind, tile_properties(plan, 1, p), 1, 1, p), (si, t_in, 1, nh, nw))
                continue
            eh, nh = hn
            nw0 = members[0][1]
            plans = {}

            def query(k):
                nonlocal queries
                if k not in plans:
                    plans[k] = plan_fn(kind, site, *frames[k], nh, nw0)
                    queries += 1
                return plans[k]

            def fill(a, b):    # frames a..b: equal plans at both ends hold in between (NACC is monotone in T_out)
                if b - a > 1 and _key(query(a)) == _key(query(b)):
                    for k in range(a + 1, b):
                        plans[k] = plans[a]
                elif b - a > 1:
                    fill(a, (a + b) // 2)
                    fill((a + b) // 2, b)
                else:
                    query(a), query(b)
            fill(0, len(frames) - 1)
            for k, (t_in, t_out) in enumerate(frames):
                plan = plans[k]
                if plan is None:
                    continue
                ck = (_key(plan), t_in, t_out)
                sigs = sig_cache.get(ck)
                if sigs is None:
                    sigs = sig_cache[ck] = tile_signatures(kind, plan, t_in, t_out)
                for ew, nw in members:
                    _offer(best, sigs, case_score(kind, tile_properties(plan, eh, ew), t_out, eh, ew),
                           (si, t_in, t_out, nh, nw))
    return best, queries


def _key(plan):
    return None if plan is None else tuple(plan[k] for k in SIG_FIELDS + ("TH", "tiles_w", "tiles_h"))


def case_score(kind, props, t_out, h, w):
    """The order of candidate shapes: most of tile_properties, then at least GATE3_ELEMS elements at the audit's sample
    frames (gate 3's mean of +-1/2 ulp errors has a spread of 0.29 / sqrt(n) ulp: 0.005 at 4096), then fewest output
    positions."""
    checked = min(t_out, 5) * h * w * (kind["Cout"] // kind["up_time"])
    return -sum(props), checked < GATE3_ELEMS, t_out * h * w


def _offer(best, sigs, score, shape):
    for s in sigs:
        cur = best.get(s)
        if cur is None or score < cur[0]:
            best[s] = (score, shape)


def kind_id(kind):
    """A stable name of a kind: every property but the extents."""
    k = kind
    return (f"{k['view']}:ci{k['Cin']}:co{k['Cout']}:k{''.join(map(str, k['kernel']))}"
            f":s{''.join(map(str, k['stride']))}"
            f":o{','.join(map(str, k['offset']))}:pt{k['pad_t']}:ut{k['up_time']}:r{int(k['residual'])}:c2{k['C2']}"
            f":gn{k['gn']}:b{int(k['bias'])}" + (":synthetic" if k.get("synthetic") else ""))


def sig_str(sig):
    return ",".join("-" if v is None else str(int(v)) for v in sig)


# ------------------------------------------------------------------------------------------ geometry and descriptors
def geometry(kind, site, t_in, t_out, nh, nw):
    """Shapes of one case: x (dense), the buffer y lives in and how y views it; extents from the tile extents nh, nw."""
    variant, direction, xl, yl, framed = site["where"]
    eh, ew = level_extent(variant, direction, yl, nh), level_extent(variant, direction, yl, nw)
    co = kind["Cout"]
    if kind["view"] == "flat":
        p = t_in * eh * ew
        return {"x": (1, 1, 1, p, kind["Cin"]), "buf": (1, 1, 1, p, co), "view": "dense", "y": (1, 1, 1, p, co)}
    xh = level_extent(variant, direction, xl, nh) + 2 * framed
    xw = level_extent(variant, direction, xl, nw) + 2 * framed
    ty, cy = (2 * t_out - 1, co // 2) if kind["up_time"] == 2 else (t_out, co)
    y = (1, ty, eh, ew, cy)
    if kind["view"].startswith("lattice"):
        buf = (1, ty, 2 * eh, 2 * ew, cy)
    elif kind["view"] == "ncdhw":
        buf = (1, cy, ty, eh, ew)
    else:
        buf = y
    return {"x": (1, t_in, xh, xw, kind["Cin"]), "buf": buf, "view": kind["view"], "y": y}


def y_view(buf, view):
    """y as the network views its buffer: dense, the (ph, pw) lattice of an up-sampler phase, or NCDHW."""
    if view.startswith("lattice"):
        ph, pw = int(view[-2]), int(view[-1])
        return buf[:, :, ph::2, pw::2]
    if view == "ncdhw":
        return buf.permute(0, 2, 3, 4, 1)
    return buf


def _strides(shape):
    s, out = 1, []
    for n in reversed(shape):
        out.append(s)
        s *= n
    return tuple(reversed(out))


def _t5(ptr, shape, strides):
    from cvvae_b200 import _lib as L
    return L.Tensor5(ptr, *shape, *strides)


class DescPlanner:
    """plan_fn of select(): cvvae_conv_tc_plan on a descriptor with the case's geometry and aligned dummy pointers
    (conv_tc_plan checks their alignment and stores them; nothing on the plan path dereferences them)."""

    def __init__(self, dtype_code):
        from cvvae_b200 import _lib as L
        self.L, self.lib, self.dtype_code = L, L.load(), dtype_code
        self.fields = L.CONV_TC_PLAN_EPILOGUE_FIELDS
        self.vals = (C.c_int32 * len(self.fields))()

    def desc(self, kind, site, t_in, t_out, nh, nw):
        L = self.L
        g = geometry(kind, site, t_in, t_out, nh, nw)
        d = L.ConvDesc()
        base = 1 << 32
        d.x = _t5(base, g["x"], _strides(g["x"]))
        bs = _strides(g["buf"])
        if g["view"].startswith("lattice"):
            ph, pw = int(g["view"][-2]), int(g["view"][-1])
            ptr = 2 * base + 2 * (ph * bs[2] + pw * bs[3])
            ys = (bs[0], bs[1], 2 * bs[2], 2 * bs[3], bs[4])
        elif g["view"] == "ncdhw":
            ptr, ys = 2 * base, (bs[0], bs[2], bs[3], bs[4], bs[1])
        else:
            ptr, ys = 2 * base, bs
        d.y = _t5(ptr, g["y"], ys)
        d.w = 3 * base
        d.bias = 4 * base if kind["bias"] else None
        d.residual = 5 * base if kind["residual"] else None
        d.Cout = kind["Cout"]
        d.KT, d.KH, d.KW = kind["kernel"]
        d.st, d.sh, d.sw = kind["stride"]
        d.off_t, d.off_h, d.off_w = kind["offset"]
        d.pad_t, d.pad_hw = kind["pad_t"], PAD_ZERO
        d.up_time = kind["up_time"]
        d.dtype = self.dtype_code
        d.alpha = 1.0
        if kind["gn"]:
            d.gn_stats, d.gn_groups = 6 * base, kind["gn"]
        if kind["C2"]:
            c2 = g["y"][:4] + (kind["C2"],)
            d.x2, d.w2 = _t5(7 * base, c2, _strides(c2)), 8 * base
        return d

    def __call__(self, kind, site, t_in, t_out, nh, nw):
        d = self.desc(kind, site, t_in, t_out, nh, nw)
        rc = self.lib.cvvae_conv_tc_plan(C.byref(d), self.vals, len(self.fields))
        assert rc == len(self.fields), (rc, self.lib.cvvae_last_error())
        plan = dict(zip(self.fields, list(self.vals)))
        return plan if plan["eligible"] else None


# ------------------------------------------------------------------------------------------ layer kinds of the network
class _Recording:
    """An operator set that runs its inner one and keeps the kind of every conv call (not its tensors)."""

    def __init__(self, inner):
        self.inner, self.kinds, self.ctx = inner, {}, None

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def conv(self, x, w, bias, **kw):
        self._record(x, w, bias, kw)
        return self.inner.conv(x, w, bias, **kw)

    def _record(self, x, w, bias, kw):
        if kw.get("w_per_batch") or kw.get("x_shared") or kw.get("out_f32") or kw.get("bias_along_m"):
            return                                   # the attention GEMMs
        from network_audit import view_kind
        variant, direction, n, t = self.ctx
        exts = [level_extent(variant, direction, lv, n) for lv in range(LEVELS)]
        out = kw["out"]
        kernel = tuple(kw.get("kernel", (1, 1, 1)))
        up_time = kw.get("up_time", 1)
        assert x.is_contiguous(), "conv inputs are dense channels-last tensors"
        flat = kernel == (1, 1, 1) and out.shape[1] == 1 and out.shape[2] == 1
        if flat:     # [B, 1, 1, T * H * W, C]: the level whose frames and extents give the positions
            lv = [lv for lv in range(LEVELS) if level_frames(direction, lv, t) * exts[lv] ** 2 == x.shape[3]]
            assert len(lv) == 1, (x.shape, exts, t)
            t_in = level_frames(direction, lv[0], t)
            where, frames, view = (variant, direction, lv[0], lv[0], False), (t_in, 1), "flat"
        else:
            view = view_kind(out)
            assert view in ("dense", "lattice", "ncdhw"), view
            if view == "lattice":
                row, off = out.stride(2) // 2, out.storage_offset()     # (ph, pw) of y[:, :, ph::2, pw::2]
                view += f"{off // row}{off % row // out.shape[4]}"
            yl = exts.index(out.shape[2])
            framed = x.shape[2] not in exts
            xl = exts.index(x.shape[2] - 2 * framed)
            t_out = (out.shape[1] + 1) // 2 if up_time == 2 else out.shape[1]
            where, frames = (variant, direction, xl, yl, framed), (x.shape[1], t_out)
        kind = {"view": view, "Cin": x.shape[4], "Cout": w.shape[1], "kernel": kernel,
                "stride": tuple(kw.get("stride", (1, 1, 1))), "offset": tuple(kw.get("offset", (0, 0, 0))),
                "pad_t": kw.get("pad_t", PAD_ZERO), "up_time": up_time, "residual": kw.get("residual") is not None,
                "C2": kw["sc_x"].shape[4] if kw.get("sc_w") is not None else 0,
                "gn": kw.get("gn_groups", 32) if kw.get("gn_stats") is not None else 0, "bias": bias is not None}
        assert kw.get("pad_hw", PAD_ZERO) == PAD_ZERO and w.shape[2] == x.shape[4] and not kw.get("w_ld")
        k = self.kinds.setdefault(kind_id(kind), dict(kind, sites={}))
        k["sites"].setdefault(where, set()).add(frames)


def record_kinds(ops, dtype=torch.float16):
    """The conv kinds of sd21 and sd3 encode (1-17 frames) and decode (the latent frame counts of those) passes at
    REC_PIXELS, real widths.  Returns [kind] with kind["sites"] = [{"where": (variant, direction, x level, y level,
    x framed), "frames": {(T_in, T_out)}}]."""
    from cvvae_b200.engine import Engine, NetConfig, prepack_params
    from oracle import cvvae_oracle as O
    rec = _Recording(ops)
    for variant in ("sd21", "sd3"):
        zc = 4 if variant == "sd21" else 16
        cfg = O.VAEConfig(variant=variant, z_channels=zc)
        sd = {k: v.to(dtype).to(DEV) for k, v in O.make_state_dict(cfg, 7).items()}
        eng = Engine(NetConfig(variant=variant, z_channels=zc), prepack_params(sd, ops, dtype), rec, dtype)
        del sd
        n_lat = level_extent(variant, "enc", LEVELS - 1, REC_PIXELS)
        for t in ENC_FRAMES:
            rec.ctx = (variant, "enc", REC_PIXELS, t)
            eng.encode(torch.rand((1, 3, t, REC_PIXELS, REC_PIXELS), device=DEV).to(dtype))
        for t in sorted({eng.encoded_frames(t) for t in ENC_FRAMES}):
            rec.ctx = (variant, "dec", n_lat, t)
            eng.decode(torch.rand((1, zc, t, n_lat, n_lat), device=DEV).to(dtype))
        del eng
    kinds = []
    for kid in sorted(rec.kinds):
        k = rec.kinds[kid]
        k["sites"] = [{"where": wh, "frames": fr} for wh, fr in sorted(k["sites"].items())]
        kinds.append(k)
    return kinds


# ------------------------------------------------------------------------------------------ the space and its cases
# Synthetic kinds (API-admissible, not layers of the network): the encoder's first causal 3x3x3 conv (128 channels, the
# pixel level, where the TW = 64 / 128 plans with 3- and 2-slot A rings occur) with a fused 1x1 shortcut of 128 / 64
# channels.  9 * 2 + 2 = 20 slabs leave the epilogue's second staging block in slot 3 of a 3-slot ring, 19 slabs in
# slot 2 of a 2-slot ring.  The network's 3x3x3 and 1x3x3 slab counts (a slab feeds all three row taps) are multiples
# of 9 and 3, so at NA = 3 its staging never wraps.
SYNTHETIC = {"wrap_na3": ("dense:ci128:co128:k333:s111:o-2,-1,-1:pt1:ut1:r0:c20:gn32:b1", 128),
             "wrap_na2": ("dense:ci128:co128:k333:s111:o-2,-1,-1:pt1:ut1:r0:c20:gn32:b1", 64)}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_plan_space_132.json")
FROZEN_SMS = 132
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}
_RECORD = {}


def build_space(ops, plan_fn):
    """Kinds (network and synthetic), and one case per reachable (kind, signature): {(kind id, signature): (kind,
    shape)}, with the enumeration's plan queries and host time."""
    kinds = record_kinds(ops)
    by_id = {kind_id(k): k for k in kinds}
    for base, c2 in SYNTHETIC.values():
        kinds.append(dict(by_id[base], C2=c2, synthetic=True))
    t0 = time.perf_counter()
    cases, queries = {}, 0
    for k in kinds:
        best, q = select(k, plan_fn)
        queries += q
        for sig, (_, shape) in best.items():
            cases[(kind_id(k), sig)] = (k, shape)
    return kinds, cases, queries, time.perf_counter() - t0


def reachable_strings(cases):
    return sorted(f"{kid}|{sig_str(sig)}" for kid, sig in cases)


def wrap_coverage(cases):
    """{NA: sorted wrap states} over the TMA-epilogue signatures."""
    seen = {}
    for _, sig in cases:
        if sig[SIG_FIELDS.index("tma_epilogue")]:
            seen.setdefault(sig[SIG_FIELDS.index("NA")], set()).add(sig[-1])
    return {na: sorted(v) for na, v in sorted(seen.items())}


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "conv_plan_space.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True, default=str)


@pytest.fixture(scope="module")
def space():
    from cvvae_b200 import _lib as L
    from cvvae_b200.ops import CudaOps
    t0 = time.perf_counter()
    kinds, cases, queries, host_s = build_space(CudaOps(), DescPlanner(L.F16))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    _RECORD["enumeration"] = {"sms": sms, "kinds": len(kinds), "plan_queries": queries, "enumeration_host_s": host_s,
                              "setup_s": time.perf_counter() - t0, "reachable": len(cases),
                              "signatures": sorted({sig_str(s) for _, s in cases}),
                              "wrap_coverage": wrap_coverage(cases),
                              "reachable_set": reachable_strings(cases)}
    _dump()
    return {"kinds": kinds, "cases": cases, "sms": sms}


def test_reachable_plan_set(space):
    """Every NA of a TMA-epilogue plan runs wrapping and non-wrapping staging; on 132 SMs the set is the frozen one."""
    cases = space["cases"]
    cov = wrap_coverage(cases)
    assert cov and all(v == [False, True] for v in cov.values()), cov
    if space["sms"] == FROZEN_SMS:
        with open(GOLDEN) as f:
            frozen = json.load(f)["reachable"]
        got = reachable_strings(cases)
        assert got == frozen, {"new": sorted(set(got) - set(frozen))[:20], "gone": sorted(set(frozen) - set(got))[:20]}


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g) * 2 - 1) * scale).to(dtype).to(DEV)


@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_every_reachable_signature_against_fp64(space, dt, monkeypatch):
    """One case per (kind, signature), through AuditOps; 16-bit also bit-identical across the three epilogues."""
    from cvvae_b200 import _lib as L
    from cvvae_b200.ops import CudaOps
    from network_audit import AuditOps, same_bits, sample_frames
    ops, dtype = CudaOps(), DTYPES[dt]
    audit = AuditOps(ops)
    planner = DescPlanner(L.F16)     # the enumeration's (16-bit) plans; fp32 runs the same shapes
    shapes = {}
    for (kid, sig), (kind, shape) in sorted(space["cases"].items(), key=lambda c: (c[0][0], sig_str(c[0][1]))):
        shapes.setdefault((kid, shape), (kind, []))[1].append(sig)
    rows, failed = [], []
    for n, ((kid, shape), (kind, sigs)) in enumerate(sorted(shapes.items(), key=lambda c: (c[0][0], c[0][1]))):
        t0 = time.perf_counter()
        si, t_in, t_out, nh, nw = shape
        site = kind["sites"][si]
        g = geometry(kind, site, t_in, t_out, nh, nw)
        # the plan is per sample (the same for any batch): a case with few elements at the audit's sample frames runs
        # as a batch, so that gate 3 averages over at least GATE3_ELEMS of them
        per_sample = len(sample_frames(t_out)) * math.prod(g["y"][2:]) * (2 if kind["up_time"] == 2 else 1)
        batch = -(-GATE3_ELEMS // per_sample)
        g = {k: ((batch,) + v[1:] if k != "view" else v) for k, v in g.items()}
        seed = 1000 * n
        taps = math.prod(kind["kernel"])
        x = _rand(g["x"], dtype, seed)
        w = _rand((taps, kind["Cout"], kind["Cin"]), dtype, seed + 1, scale=2 * (taps * kind["Cin"]) ** -0.5)
        bias = _rand((kind["Cout"],), torch.float32, seed + 2, 0.3) if kind["bias"] else None
        kw = dict(kernel=kind["kernel"], stride=kind["stride"], offset=kind["offset"], pad_t=kind["pad_t"],
                  pad_hw=PAD_ZERO, up_time=kind["up_time"])
        if kind["residual"]:
            kw["residual"] = _rand(g["y"], dtype, seed + 3)
        if kind["C2"]:
            kw["sc_x"] = _rand(g["y"][:4] + (kind["C2"],), dtype, seed + 4)
            kw["sc_w"] = _rand((kind["Cout"], kind["C2"]), dtype, seed + 5, scale=kind["C2"] ** -0.5)

        def launch(odd, tma):
            """A NaN-filled output of the kind's view (odd: one element past an aligned start), its statistics, plan."""
            monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1" if tma else "0")
            buf = torch.full((math.prod(g["buf"]) + odd,), float("nan"), dtype=dtype, device=DEV)[odd:].view(g["buf"])
            y = y_view(buf, g["view"])
            skw = dict(gn_stats=ops.new_stats(batch, kind["gn"], DEV), gn_groups=kind["gn"]) if kind["gn"] else {}
            return y, skw, ops.conv_tc_plan(x, w, bias, out=y, epilogue=True, **kw, **skw)

        y, skw, plan = launch(0, True)
        audit.conv(x, w, bias, out=y, **kw, **skw)
        arow = audit.rows[-1]
        bad = list(arow["failed"])
        # the shape reaches its signatures: the plan of the real tensors is the enumerated one
        want = planner(kind, site, t_in, t_out, nh, nw)
        if dtype != torch.float32 and any(plan[k] != want[k] for k in want if k != "grid"):
            bad.append(f"plan of the tensors {plan} differs from the enumerated {want}")
        if plan["eligible"] != 1:
            bad.append(f"not on the tensor-core path: {plan}")
        elif dtype != torch.float32:
            missing = [s for s in sigs if s not in tile_signatures(kind, plan, t_in, t_out)]
            if missing:
                bad.append(f"signatures not reached: {[sig_str(s) for s in missing]}")
        row = {"kind": kid, "signatures": [sig_str(s) for s in sigs], "where": site["where"], "T_in": t_in,
               "T_out": t_out, "tile": [nh, nw], "x": g["x"], "y": g["y"], "view": g["view"], "plan": plan,
               "partial_ragged_interior": tile_properties(plan, g["y"][2], g["y"][3]) if plan["eligible"] else None}
        row.update({k: arow[k] for k in ("worst_bound_ratio", "correctly_rounded_share", "mean_signed_ulp",
                                         "stats_max_abs_err", "frames_checked") if k in arow})
        if dtype != torch.float32:
            # the register epilogue, and the general loop into an odd-offset output: the same bits
            y_reg, skw_reg, plan_reg = launch(0, False)
            ops.conv(x, w, bias, out=y_reg, **kw, **skw_reg)
            y_odd, skw_odd, plan_odd = launch(1, True)
            ops.conv(x, w, bias, out=y_odd, **kw, **skw_odd)
            torch.cuda.synchronize()
            if plan_reg["tma_epilogue"] or plan_odd["tma_epilogue"] or plan_odd["vec2"]:
                bad.append(f"epilogue switches not taken: register {plan_reg}, odd {plan_odd}")
            eq = {"register": same_bits(y, y_reg), "odd_offset": same_bits(y, y_odd)}
            if kind["gn"]:
                eq["register_stats"] = torch.equal(skw["gn_stats"], skw_reg["gn_stats"])
                eq["odd_offset_stats"] = torch.equal(skw["gn_stats"], skw_odd["gn_stats"])
            row["bit_equal"] = eq
            bad += [f"{k}: not bit-identical to the TMA-epilogue run" for k, v in eq.items() if not v]
            del y_reg, y_odd
        monkeypatch.delenv("CVVAE_TMA_EPILOGUE", raising=False)
        row["failed"] = bad
        row["wall_s"] = round(time.perf_counter() - t0, 4)
        rows.append(row)
        if bad:
            failed.append({k: row[k] for k in ("kind", "signatures", "where", "T_in", "tile", "failed")})
        audit.rows.clear()
        del x, w, y, kw
    _RECORD[dt] = {"cases": len(rows), "failures": failed, "rows": rows}
    _dump()
    assert not failed, failed[:10]
    covered = {(r["kind"], s) for r in rows for s in r["signatures"]}
    assert covered == {(kid, sig_str(sig)) for kid, sig in space["cases"]}
