"""The fp32 oracle's Conv2d with the un-merged LoRA of a LoCon adapter, as peft's lora.Conv2d computes it [3P, restated:
diffusers / peft are not importable here, so there is no golden from the reference]: a k x k `down` conv with the base
conv's stride and padding, a 1x1 `up` conv, times the scale.  Un-merged on purpose: the CUDA path merges the delta into
the weight, so the two sides reach it by different routes.  oracle/unet.py applies `Ctx.lora` in its linear helper only
(time_emb_proj goes through that one); the `locon_oracle` fixture puts this conv in place of the oracle's for a test."""
import pytest
import torch.nn.functional as F

from oracle import unet as ou


def conv(c: ou.Ctx, name: str, x, stride=1, padding=1):
    """oracle.unet.conv + s * up_1x1(down_kxk(x)) for every (A [r, in, k, k], B [out, r], s) of c.lora[name]."""
    y = F.conv2d(x, c.w(name + ".weight"), c.w(name + ".bias") if c.has(name + ".bias") else None, stride=stride,
                 padding=padding)
    for A, Bm, s in c.lora.get(name, ()):
        y = y + s * F.conv2d(F.conv2d(x, A, stride=stride, padding=A.shape[-1] // 2), Bm[:, :, None, None])
    return y


@pytest.fixture(autouse=True)
def locon_oracle(monkeypatch):
    """Every oracle forward of the importing test module applies conv LoRA entries of its Ctx (resnet, the samplers and
    unet_forward look `conv` up in oracle.unet when they run)."""
    monkeypatch.setattr(ou, "conv", conv)
