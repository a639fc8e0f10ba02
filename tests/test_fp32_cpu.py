"""float32 (CVVAE_F32) plumbing without a GPU: dtype codes, header / binding agreement, the CPU model error, video_io's
refusal of fp32."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dtype_code_maps_float32_to_f32():
    from cvvae_b200 import _lib as L
    from cvvae_b200.ops import dtype_code
    assert (L.F16, L.BF16, L.F32) == (0, 1, 2)
    assert dtype_code(torch.float32) == L.F32
    assert dtype_code(torch.float16) == L.F16 and dtype_code(torch.bfloat16) == L.BF16
    with pytest.raises(L.CvvaeError):
        dtype_code(torch.float64)


def test_header_enum_and_abi_version_agree_with_binding():
    from cvvae_b200 import _lib as L
    src = open(os.path.join(ROOT, "include", "cvvae_b200.h")).read()
    enum = re.search(r"enum\s*\{\s*CVVAE_F16\s*=\s*(\d+),\s*CVVAE_BF16\s*=\s*(\d+),\s*CVVAE_F32\s*=\s*(\d+)\s*\}", src)
    assert enum and tuple(int(v) for v in enum.groups()) == (L.F16, L.BF16, L.F32)
    ver = re.search(r"#define\s+CVVAE_ABI_VERSION\s+(\d+)", src)
    assert ver and int(ver.group(1)) == L.ABI_VERSION == 3


def test_float32_model_on_cpu_raises_the_cuda_error():
    from cvvae_b200 import CVVAEModel
    m = CVVAEModel(ch=32)
    assert next(m.parameters()).dtype == torch.float32
    with pytest.raises(RuntimeError, match="runs on CUDA"):
        m.encode(torch.zeros((1, 3, 1, 16, 16)))


def test_video_io_rejects_f32():
    """The video_io entry points are 16-bit only: CVVAE_F32 is an argument error with a message, before any launch."""
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    fake = 256   # never dereferenced: the dtype check precedes every launch
    for rc in (lib.cvvae_video_u8_to_f16(fake, fake, 1, 2, 2, L.F32, None),
               lib.cvvae_video_f16_to_u8(fake, fake, 1, 2, 2, L.F32, None),
               lib.cvvae_video_resize_u8(fake, fake, None, 1, 4, 4, 2, 2, L.F32, None)):
        assert rc == -1
        assert b"float16 / bfloat16 only" in lib.cvvae_last_error()
