"""Zero-edit drop-in (north_star: "cvvae_inference_video.py and the SD pipelines call it unchanged").

With `compat/` in front of sys.path, the reference inference script's `from models.modeling_vae import CVVAEModel`
resolves to this package.  The call sequence of that script (cvvae_inference_video.py) is replayed here; the engine runs
on the CPU test double of the operator set (tests/fake_ops.py) and `.cuda()` is a no-op - what is checked is the
host-side contract: from_pretrained(path, subfolder=, torch_dtype=), requires_grad_, the fp16 input convention,
encode(...).latent_dist.sample(), decode(...).sample, shapes and value range.
"""
import importlib
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def compat_path(monkeypatch):
    monkeypatch.syspath_prepend(os.path.join(ROOT, "compat"))
    for name in [n for n in sys.modules if n == "models" or n.startswith("models.") or n.startswith("diffuser_engine")]:
        monkeypatch.delitem(sys.modules, name)
    yield


def test_compat_paths_resolve_to_the_engine(compat_path):
    import cvvae_b200
    m1 = importlib.import_module("models.modeling_vae")
    m2 = importlib.import_module("diffuser_engine.models.modeling_vae")
    assert m1.CVVAEModel is cvvae_b200.CVVAEModel and m1.CVVAESD3Model is cvvae_b200.CVVAESD3Model
    assert m2.CVVAEModel is cvvae_b200.CVVAEModel


def test_inference_script_call_sequence(compat_path, monkeypatch, tmp_path):
    """The calls the reference's inference script makes, in its order, through the `models.modeling_vae` import path."""
    from fake_ops import FakeOps
    from oracle import cvvae_oracle as O
    from torchvision import transforms
    import cvvae_b200
    # a small "published checkpoint": config.json + safetensors under <path>/vae3d, as the script expects
    wrap = dict(tile_spatial_size=72, en_de_n_frames_a_time=4)
    m = cvvae_b200.CVVAEModel(ch=32, **wrap)
    m.load_state_dict(O.make_state_dict(O.VAEConfig(variant="sd21", ch=32, **wrap), 1234))
    m.save_pretrained(str(tmp_path / "ckpt" / "vae3d"))
    monkeypatch.setattr(cvvae_b200.modeling_vae._CVVAEBase, "_ops_factory", FakeOps)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.nn.Module, "cuda", lambda self, *a, **k: self)
    torch.manual_seed(0)
    CVVAEModel = importlib.import_module("models.modeling_vae").CVVAEModel
    assert CVVAEModel is cvvae_b200.CVVAEModel
    vae = CVVAEModel.from_pretrained(str(tmp_path / "ckpt"), subfolder="vae3d", torch_dtype=torch.float16)
    vae.requires_grad_(False)
    vae = vae.cuda()
    # a decoded clip: 7 uint8 frames [T, H, W, C] -> resized [T, C, H, W] -> [1, C, T, H, W] fp16 in [-1, 1]
    n_frames, H0, W0 = 7, 60, 90
    g = torch.Generator().manual_seed(3)
    frames = torch.randint(0, 256, (n_frames, H0, W0, 3), generator=g, dtype=torch.uint8)
    video = transforms.Resize(size=(80, 104))(frames.permute(0, 3, 1, 2))
    video = video.permute(1, 0, 2, 3).unsqueeze(0).half()
    frame_end = 1 + (n_frames - 1) // 4 * 4
    video = (video / 127.5 - 1.0)[:, :, :frame_end].cuda()
    latent = vae.encode(video).latent_dist.sample()
    assert tuple(latent.shape) == (1, 4, 2, 10, 13) and latent.dtype == torch.float16
    results = vae.decode(latent).sample
    results = results.squeeze(0).permute(1, 2, 3, 0)
    arr = ((torch.clamp(results, -1.0, 1.0) + 1.0) * 127.5).to("cpu", dtype=torch.uint8)
    assert arr.dtype == torch.uint8 and tuple(arr.shape) == (5, 80, 104, 3)
    assert 0 < arr.float().mean().item() < 255
