"""Drop-in ``CVVAEModel`` / ``CVVAESD3Model``: the reference's Python surface over the sm_90a engine.

Mirrors models/modeling_vae.py of the reference - same constructor keyword arguments and defaults
(:23-51, :347-381), ``config`` attribute/dict access, ``from_pretrained(path, subfolder=, torch_dtype=)``
reading ``config.json`` + ``diffusion_pytorch_model.safetensors``, ``encode()`` / ``decode()`` /
``forward()`` signatures and return objects (:114-142, :212-228, :298-319), 4-D input handling, and the
exact temporal-chunk (:193-210, :279-296) / spatial-tile (:144-191, :230-277) / in-place linear blend
(:321-341) decomposition, which is part of the function being computed (GroupNorm statistics are per
chunk x tile).  ``cvvae_inference_video.py`` and the SD pipelines call it unchanged.

The arithmetic runs in hand-written CUDA (cvvae_b200/csrc) through the C ABI; this file holds no
PyTorch compute beyond slicing / concatenation of tile results and the tiny posterior helpers.
"""
from __future__ import annotations

import inspect
import json
import math
import os
import weakref
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import torch
import torch.nn as nn

from .engine import Engine, NetConfig, prepack_params
from .params import ParamTree, build_param_tree, param_shapes


class FrozenConfig(dict):
    """``model.config.key`` and ``model.config["key"]`` (diffusers FrozenDict behaviour)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


@dataclass
class DecoderOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


@dataclass
class AutoencoderKLOutput:
    latent_dist: "DiagonalGaussianDistribution"

    def __getitem__(self, i):
        return (self.latent_dist,)[i]


class DiagonalGaussianDistribution:
    """Posterior wrapper (diffusers' class; reference twin lvdm/modules/distributions/distributions.py:24-73)."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        # diffusers.utils.randn_tensor semantics: a CPU generator draws on the CPU and the noise is moved (pipelines
        # commonly pass CPU generators for reproducibility across devices); otherwise draw on the tensor's device
        dev = self.parameters.device
        gdev = generator.device if generator is not None else dev
        if gdev.type != dev.type:
            eps = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.parameters.dtype).to(dev)
        else:
            eps = torch.randn(self.mean.shape, generator=generator, device=dev, dtype=self.parameters.dtype)
        return self.mean + self.std * eps

    def mode(self) -> torch.Tensor:
        return self.mean


def _register_config(init):
    """Record constructor kwargs (with defaults) like diffusers' @register_to_config."""
    sig = inspect.signature(init)

    def wrapper(self, *args, **kwargs):
        bound = sig.bind(self, *args, **kwargs)
        bound.apply_defaults()
        cfg = {k: v for k, v in bound.arguments.items() if k != "self"}
        nn.Module.__init__(self)
        object.__setattr__(self, "_config", FrozenConfig(cfg))
        init(self, *args, **kwargs)

    wrapper.__signature__ = sig
    wrapper.__doc__ = init.__doc__
    return wrapper


class _NetHandle(ParamTree):
    """`model.encoder` / `model.decoder`: parameter owner + callable that runs the CUDA engine."""

    def __init__(self, owner: nn.Module, which: str):
        super().__init__()
        object.__setattr__(self, "_owner_ref", weakref.ref(owner))
        self._which = which

    def forward(self, x: torch.Tensor, **unused) -> torch.Tensor:
        return self._owner_ref()._run_net(self._which, x)


class _CVVAEBase(nn.Module):
    config_name = "config.json"
    weights_name = "diffusion_pytorch_model.safetensors"
    _ops_factory = None  # tests may inject a CPU restatement of the operator set; production leaves None
    max_tiles_per_batch = 2  # equally shaped spatial tiles run through the network together (activation memory x2)

    # ---- construction helpers -------------------------------------------------
    def _setup(self, net: NetConfig, en_de_n_frames_a_time, time_n_compress, spatial_n_compress, tile_spatial_size,
               num_video_frames, tile_overlap_ratio, reshape_z_dim_to_4, reshape_x_dim_to_4):
        self.net = net
        # `self.encoder(tile)` / `self.decoder(tile)` stay callable: the operator seam of the reference
        # (modeling_vae.py:162,249).  The handles own the parameters under the reference's key names.
        self.add_module("encoder", _NetHandle(self, "encode"))
        self.add_module("decoder", _NetHandle(self, "decode"))
        build_param_tree(self, param_shapes(net))
        # derived attributes: modeling_vae.py:84-112
        if en_de_n_frames_a_time is not None:
            assert time_n_compress is not None
            assert en_de_n_frames_a_time % time_n_compress == 0
            self.encode_n_frames_a_time = en_de_n_frames_a_time
            self.decode_n_frames_a_time = en_de_n_frames_a_time // time_n_compress
        else:
            self.encode_n_frames_a_time = None
            self.decode_n_frames_a_time = None
        if num_video_frames is not None:
            assert time_n_compress is not None
            self.num_video_frames = num_video_frames
            self.num_latent_frames = 1 + (num_video_frames - 1) // time_n_compress
        else:
            self.num_video_frames = None
            self.num_latent_frames = None
        if tile_spatial_size is not None:
            assert spatial_n_compress is not None and tile_overlap_ratio is not None
            self.pixel_tile_size = tile_spatial_size
            self.latent_tile_size = tile_spatial_size // spatial_n_compress
            self.tile_overlap_ratio = tile_overlap_ratio
        else:
            self.pixel_tile_size = None
            self.latent_tile_size = None
            self.tile_overlap_ratio = None
        self.reshape_z_dim_to_4 = reshape_z_dim_to_4
        self.reshape_x_dim_to_4 = reshape_x_dim_to_4
        self._engine_cache = None
        self._graphs_enabled = False
        self._graph_cache = {}
        self._graph_pool = None
        self._graph_max = 8
        self._tile_runner = None   # parallel.UnitShardedVAE installs its distributed tile loop here
        self.requires_grad_(False)
        self.eval()

    @property
    def config(self) -> FrozenConfig:
        return self._config

    @property
    def dtype(self) -> torch.dtype:
        return next(self.parameters()).dtype

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    # ---- checkpoint I/O (diffusers ModelMixin surface used by the reference scripts) ----------
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None,
                        torch_dtype: Optional[torch.dtype] = None, **unused):
        d = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else pretrained_model_name_or_path
        with open(os.path.join(d, cls.config_name)) as f:
            raw = json.load(f)
        accepted = set(inspect.signature(cls.__init__).parameters) - {"self"}
        cfg = {k: v for k, v in raw.items() if k in accepted}
        model = cls(**cfg)
        st = os.path.join(d, cls.weights_name)
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(d, "diffusion_pytorch_model.bin"), map_location="cpu")
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model

    def save_pretrained(self, save_directory: str):
        from safetensors.torch import save_file
        os.makedirs(save_directory, exist_ok=True)
        cfg = dict(self.config)
        cfg["_class_name"] = type(self).__name__
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        save_file({k: v.contiguous() for k, v in self.state_dict().items()}, os.path.join(save_directory, self.weights_name))

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        self._engine_cache = None
        self._graph_cache = {}
        # the sd3 reference registers the same down-sampler conv under two names in some diffusers versions;
        # tolerate the alias when present
        sd = {k: v for k, v in state_dict.items() if ".Conv2d_0." not in k}
        return super().load_state_dict(sd, strict=strict, assign=assign)

    def _apply(self, fn, *a, **k):
        self._engine_cache = None
        self._graph_cache = {}
        return super()._apply(fn, *a, **k)

    # ---- engine ---------------------------------------------------------------
    def _engine(self) -> Engine:
        p0 = next(self.parameters())
        # parameter versions: in-place updates after the first call (param.data.copy_, weight merging, optimiser steps)
        # must re-pack the weights, as the reference modules would simply see the new values
        key = (p0.device, p0.dtype, sum(p._version for p in self.parameters()))
        if self._engine_cache is None or self._engine_cache[0] != key:
            self._graph_cache = {}
            if self._ops_factory is not None:
                ops = self._ops_factory()
            else:
                if p0.device.type != "cuda":
                    raise RuntimeError("cvvae_b200 runs on CUDA (sm_90a) only: move the model with .cuda(); "
                                       "there is no CPU or PyTorch fallback path")
                if p0.dtype not in (torch.float16, torch.bfloat16, torch.float32):
                    raise RuntimeError(f"cvvae_b200 computes in float16, bfloat16 or float32; model dtype is {p0.dtype}")
                from .ops import CudaOps
                ops = CudaOps()
            packed = prepack_params(self.state_dict(), ops, p0.dtype)
            self._engine_cache = (key, Engine(self.net, packed, ops, p0.dtype))
        return self._engine_cache[1]

    def invalidate_weights(self):
        """Drop the pre-packed weights and captured graphs (call after writing parameters through `.data`, which the
        version check in `_engine` cannot see)."""
        self._engine_cache = None
        self._graph_cache = {}
        return self

    def enable_cuda_graphs(self, enabled: bool = True, max_cached: int = 8):
        """Replay each network call (one encoder / decoder pass over a tile batch) as a captured CUDA graph.

        The chunk/tile work list of one clip launches ~600 kernels per tile; at small tiles (image path, 256^2 clips,
        the 72^2 mid-block) the host cannot issue them as fast as the GPU retires them.  One graph is captured per
        (direction, input shape) on first use - `max_cached` of them are kept, sharing one memory pool - and later
        calls copy the input into the graph's static buffer and replay.  Results are identical to the eager path
        (same kernels, same order).  (SURVEY.md section 8f row 1.)
        """
        self._graphs_enabled = bool(enabled)
        self._graph_max = int(max_cached)
        if not enabled:
            self._graph_cache = {}
        return self

    def _run_net_eager(self, eng: Engine, which: str, x: torch.Tensor) -> torch.Tensor:
        return eng.encode(x) if which == "encode" else eng.decode(x)

    def _run_net(self, which: str, x: torch.Tensor) -> torch.Tensor:
        self._check_input(x)
        if x.is_cuda and x.device.index != torch.cuda.current_device():
            with torch.cuda.device(x.device):   # kernels, streams and graph capture belong to the model's device
                return self._run_net(which, x)
        eng = self._engine()
        if (not self._graphs_enabled or self._ops_factory is not None or getattr(eng.ops, "profile", None) is not None
                or torch.cuda.is_current_stream_capturing()):
            return self._run_net_eager(eng, which, x)
        key = (which, tuple(x.shape))
        entry = self._graph_cache.get(key)
        if entry is None:
            static_in = x.detach().clone(memory_format=torch.contiguous_format)
            cur = torch.cuda.current_stream(x.device)
            side = torch.cuda.Stream(device=x.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):               # one eager pass first: module loading, func attributes, allocator warm-up
                self._run_net_eager(eng, which, static_in)
            cur.wait_stream(side)
            if self._graph_pool is None:
                self._graph_pool = torch.cuda.graph_pool_handle()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=self._graph_pool):
                static_out = self._run_net_eager(eng, which, static_in)
            while len(self._graph_cache) >= max(1, self._graph_max):
                self._graph_cache.pop(next(iter(self._graph_cache)))
            entry = self._graph_cache[key] = (graph, static_in, static_out)
        graph, static_in, static_out = entry
        static_in.copy_(x)
        graph.replay()
        return static_out.clone()

    def _check_input(self, x):
        if x.dtype != self.dtype:
            raise RuntimeError(f"Input type ({x.dtype}) and model weight type ({self.dtype}) should be the same")
        if x.device != self.device:
            raise RuntimeError(f"Input device ({x.device}) and model device ({self.device}) should be the same")

    # ---- forward: modeling_vae.py:114-142 ---------------------------------------
    @torch.no_grad()
    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True,
                generator: Optional[torch.Generator] = None, num_frames: int = None):
        posterior = self.encode(sample).latent_dist
        z = posterior.sample(generator=generator) if sample_posterior else posterior.mode()
        dec = self.decode(z, num_frames=num_frames).sample
        if not return_dict:
            return (dec,)
        return DecoderOutput(sample=dec)

    # ---- tiling: modeling_vae.py:144-191, 230-277 -------------------------------
    def _blend_v(self, a: torch.Tensor, b: torch.Tensor, overlap: int) -> torch.Tensor:
        self._engine().ops.blend(a.permute(0, 2, 3, 4, 1), b.permute(0, 2, 3, 4, 1), overlap, 1)
        return b

    def _blend_h(self, a: torch.Tensor, b: torch.Tensor, overlap: int) -> torch.Tensor:
        self._engine().ops.blend(a.permute(0, 2, 3, 4, 1), b.permute(0, 2, 3, 4, 1), overlap, 0)
        return b

    # public names of the reference (:321-341)
    def blend_h(self, a, b, overlap_size):
        return self._blend_h(a, b, overlap_size)

    def blend_v(self, a, b, overlap_size):
        return self._blend_v(a, b, overlap_size)

    def _tile_rows(self, x: torch.Tensor, fn, in_tile: int, out_tile: int):
        """Run `fn` over the spatial tiles of one temporal chunk and blend them in place, in the reference's order.
        Returns (rows of blended tiles, stride of the kept window of every tile but the last of a row / column)."""
        ratio = self.tile_overlap_ratio
        in_stride = round(in_tile * (1 - ratio))
        out_overlap = round(out_tile * ratio)
        out_stride = out_tile - out_overlap
        # tile windows in the reference's order; equally shaped tiles are pushed through the network as one batch
        # (tiles are independent encoder/decoder calls - GroupNorm statistics are per sample - so this is the same
        # arithmetic with half the launches and better-filled grids on the low-resolution layers)
        windows = []
        for i in range(0, x.shape[3], in_stride):
            row = []
            for j in range(0, x.shape[4], in_stride):
                row.append((i, j))
                if j + in_tile >= x.shape[4]:
                    break
            windows.append(row)
            if i + in_tile >= x.shape[3]:
                break
        flat = [(r, c, x[:, :, :, i:i + in_tile, j:j + in_tile]) for r, row in enumerate(windows) for c, (i, j) in enumerate(row)]
        results = (self._tile_runner or self._run_tiles_local)(flat, fn)
        rows = [[results[(r, c)] for c in range(len(row))] for r, row in enumerate(windows)]
        # blend against the already blended upper / left neighbours, in place (reference order)
        for i, cols in enumerate(rows):
            for j, tile in enumerate(cols):
                if i > 0:
                    self._blend_v(rows[i - 1][j], tile, out_overlap)
                if j > 0:
                    self._blend_h(cols[j - 1], tile, out_overlap)
        return rows, out_stride

    def _run_tiles_local(self, flat, fn):
        """flat = [(row, col, tile view)] -> {(row, col): network output}; equally shaped neighbours share a batch."""
        results = {}
        if not flat:
            return results
        B = flat[0][2].shape[0]
        k = 0
        while k < len(flat):
            group = [flat[k]]
            while (len(group) < self.max_tiles_per_batch and k + len(group) < len(flat)
                   and flat[k + len(group)][2].shape == flat[k][2].shape):
                group.append(flat[k + len(group)])
            if len(group) == 1:
                results[(group[0][0], group[0][1])] = fn(group[0][2])
            else:
                out = fn(torch.cat([g[2] for g in group], dim=0))
                for n, g in enumerate(group):
                    results[(g[0], g[1])] = out[n * B:(n + 1) * B]
            k += len(group)
        return results

    def _assemble(self, rows, out_stride: int, dst: torch.Tensor, t_src0: int = 0) -> None:
        """Copy the kept window of every blended tile into its place of the pre-allocated result `dst`
        ([B, C, T, H, W]; frames `t_src0:` of the tiles) - one strided copy kernel per tile instead of the reference's
        crop + cat over columns + cat over rows (+ cat over chunks)."""
        ops = self._engine().ops
        y0 = 0
        for i, cols in enumerate(rows):
            x0 = 0
            h = out_stride if i < len(rows) - 1 else cols[0].shape[3]
            for j, tile in enumerate(cols):
                w = out_stride if j < len(cols) - 1 else tile.shape[4]
                src = tile[:, :, t_src0:, :h, :w]
                ops.copy(src.permute(0, 2, 3, 4, 1), dst[:, :, :, y0:y0 + h, x0:x0 + w].permute(0, 2, 3, 4, 1))
                x0 += w
            y0 += h

    @staticmethod
    def _assembled_hw(rows, out_stride: int) -> Tuple[int, int]:
        hh = out_stride * (len(rows) - 1) + rows[-1][0].shape[3]
        ww = out_stride * (len(rows[0]) - 1) + rows[0][-1].shape[4]
        return hh, ww

    def _spatial_tiled(self, x: torch.Tensor, fn, in_tile: Optional[int], out_tile: Optional[int]) -> torch.Tensor:
        if in_tile is None:
            return fn(x)
        rows, out_stride = self._tile_rows(x, fn, in_tile, out_tile)
        if len(rows) == 1 and len(rows[0]) == 1:
            return rows[0][0]
        t0 = rows[0][0]
        hh, ww = self._assembled_hw(rows, out_stride)
        out = torch.empty((t0.shape[0], t0.shape[1], t0.shape[2], hh, ww), dtype=t0.dtype, device=t0.device)
        self._assemble(rows, out_stride, out)
        return out

    def spatial_tiled_encode(self, x):
        return self._spatial_tiled(x, self.encoder, self.pixel_tile_size, self.latent_tile_size)

    def spatial_tiled_decode(self, z, **kwargs):
        return self._spatial_tiled(z, self.decoder, self.latent_tile_size, self.pixel_tile_size)

    # ---- chunking: modeling_vae.py:193-210, 279-296 ---------------------------------
    @staticmethod
    def _chunks(n_frames: int, stride: int):
        n_rounds = math.ceil((n_frames - 1) / stride)
        n_rounds = 1 if n_rounds == 0 else n_rounds
        return [(n * stride, (n + 1) * stride + 1) for n in range(n_rounds)]

    def _chunked(self, x: torch.Tensor, fn, stride: Optional[int], in_tile: Optional[int], out_tile: Optional[int],
                 out_frames) -> torch.Tensor:
        """Temporal chunk loop x spatial tile loop of the reference, every (chunk, tile) result written ONCE into the
        pre-allocated output: chunk n > 0 drops its first output frame (modeling_vae.py:204-206, 290-292)."""
        if stride is None:
            return self._spatial_tiled(x, fn, in_tile, out_tile)
        assert x.dim() == 5
        chunks = self._chunks(x.shape[2], stride)
        if len(chunks) == 1:
            return self._spatial_tiled(x[:, :, chunks[0][0]:chunks[0][1]], fn, in_tile, out_tile)
        lens = [out_frames(min(b, x.shape[2]) - a) - (1 if n else 0) for n, (a, b) in enumerate(chunks)]
        out, t = None, 0
        for n, (a, b) in enumerate(chunks):
            xc = x[:, :, a:b]
            if in_tile is None:
                r = fn(xc)
                rows, ostride = [[r]], r.shape[3]
            else:
                rows, ostride = self._tile_rows(xc, fn, in_tile, out_tile)
            t0 = rows[0][0]
            if out is None:
                hh, ww = self._assembled_hw(rows, ostride)
                out = torch.empty((t0.shape[0], t0.shape[1], sum(lens), hh, ww), dtype=t0.dtype, device=t0.device)
            assert t0.shape[2] - (1 if n else 0) == lens[n], (t0.shape, lens, n)
            self._assemble(rows, ostride, out[:, :, t:t + lens[n]], 1 if n else 0)
            t += lens[n]
        return out

    def tiled_encode(self, x):
        return self._chunked(x, self.encoder, self.encode_n_frames_a_time, self.pixel_tile_size, self.latent_tile_size,
                             self._engine().encoded_frames)

    def tiled_decode(self, z, **kwargs):
        return self._chunked(z, self.decoder, self.decode_n_frames_a_time, self.latent_tile_size, self.pixel_tile_size,
                             self._engine().decoded_frames)

    # ---- encode / decode: modeling_vae.py:212-228, 298-319 ---------------------------
    def _maybe_offload_hook(self):
        hook = getattr(self, "_hf_hook", None)  # accelerate offload hook pass-through (apply_forward_hook)
        if hook is not None and hasattr(hook, "pre_forward"):
            hook.pre_forward(self)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        self._maybe_offload_hook()
        if x.dim() == 4:
            if self.num_video_frames is not None:
                t = self.num_video_frames
                bt, c, h, w = x.shape
                x = x.reshape(bt // t, t, c, h, w).permute(0, 2, 1, 3, 4)
            else:
                x = x.unsqueeze(2)
        moments = self.tiled_encode(x)
        posterior = DiagonalGaussianDistribution(moments)
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, num_frames: int = None, return_dict: bool = True):
        self._maybe_offload_hook()
        if z.dim() == 4:
            t = num_frames if num_frames is not None else self.num_latent_frames
            if t is not None:
                bt, c, h, w = z.shape
                z = z.reshape(bt // t, t, c, h, w).permute(0, 2, 1, 3, 4)
            else:
                z = z.unsqueeze(2)
        x = self.tiled_decode(z)
        if self.reshape_x_dim_to_4:
            b, c, t, h, w = x.shape
            x = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
        if not return_dict:
            return (x,)
        return DecoderOutput(sample=x)


class CVVAEModel(_CVVAEBase):
    """SD2.1-compatible CV-VAE (4-channel latent); reference models/modeling_vae.py:20-341."""

    @_register_config
    def __init__(self, double_z=True, z_channels=4, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                 num_res_blocks=2, attn_resolutions=[], dropout=0.0, use_3d_conv=True, half_3d=True,
                 causal_encoder=True, causal_decoder=False, encoder_attn_type="vanilla-xformers",
                 decoder_attn_type="spatial-temporal-xformer", scaling_factor: float = 0.18215,
                 force_upcast: float = True, en_de_n_frames_a_time: Optional[int] = 16,
                 time_n_compress: Optional[int] = 4, spatial_n_compress: Optional[int] = 8,
                 tile_spatial_size: Optional[int] = 576, num_video_frames: Optional[int] = None,
                 tile_overlap_ratio: Optional[float] = 0.2222, reshape_z_dim_to_4: bool = False,
                 reshape_x_dim_to_4: bool = False):
        if not use_3d_conv:
            raise NotImplementedError("use_3d_conv=False is not a CV-VAE configuration (no shipped checkpoint uses it)")
        if attn_resolutions:
            raise NotImplementedError("attn_resolutions != [] is not used by any CV-VAE checkpoint")
        if dropout:
            raise NotImplementedError("dropout is a training-only setting")
        net = NetConfig(variant="sd21", in_channels=in_channels, out_ch=out_ch, z_channels=z_channels,
                        widths=tuple(ch * m for m in ch_mult), num_res_blocks=num_res_blocks, double_z=double_z,
                        causal_encoder=causal_encoder, causal_decoder=causal_decoder, half_3d=half_3d,
                        encoder_attn_type=encoder_attn_type, decoder_attn_type=decoder_attn_type)
        self._setup(net, en_de_n_frames_a_time, time_n_compress, spatial_n_compress, tile_spatial_size,
                    num_video_frames, tile_overlap_ratio, reshape_z_dim_to_4, reshape_x_dim_to_4)


class CVVAESD3Model(_CVVAEBase):
    """SD3-compatible CV-VAE (16-channel latent); reference models/modeling_vae.py:344-667."""

    @_register_config
    def __init__(self, in_channels: int = 3, out_channels: int = 16,
                 down_block_types=["DownEncoderBlock3D"] * 4, up_block_types=["UpDecoderBlock3D"] * 4,
                 block_out_channels=[128, 256, 512, 512], layers_per_block=2, norm_num_groups=32, act_fn="silu",
                 double_z=True, mid_block_add_attention=True, causal_encoder=True, causal_decoder=False,
                 half_3d=True, en_de_n_frames_a_time: Optional[int] = 16, time_n_compress: Optional[int] = 4,
                 spatial_n_compress: Optional[int] = 8, tile_spatial_size: Optional[int] = 576,
                 num_video_frames: Optional[int] = None, tile_overlap_ratio: Optional[float] = 0.2222,
                 reshape_z_dim_to_4: bool = False, reshape_x_dim_to_4: bool = False):
        if act_fn not in ("silu", "swish"):
            raise NotImplementedError(f"act_fn {act_fn!r}: CV-VAE uses SiLU")
        if any(t != "DownEncoderBlock3D" for t in down_block_types) or any(t != "UpDecoderBlock3D" for t in up_block_types):
            raise ValueError("unknown block type")
        net = NetConfig(variant="sd3", in_channels=in_channels, out_ch=in_channels, z_channels=out_channels,
                        widths=tuple(block_out_channels), num_res_blocks=layers_per_block, groups=norm_num_groups,
                        double_z=double_z, causal_encoder=causal_encoder, causal_decoder=causal_decoder,
                        half_3d=half_3d, mid_block_add_attention=mid_block_add_attention)
        self._setup(net, en_de_n_frames_a_time, time_n_compress, spatial_n_compress, tile_spatial_size,
                    num_video_frames, tile_overlap_ratio, reshape_z_dim_to_4, reshape_x_dim_to_4)
