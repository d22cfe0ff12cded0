"""SURVEY 8f-2 on the GPU: the two CLIP text towers of encode_prompt (lora_pipeline.py:315-347 -> diffusers
encode_prompt -> transformers CLIPTextModel / CLIPTextModelWithProjection [3P]) executed on this repo's kernels
(`PackedClipText`: GEMMs with bias / quick-gelu / erf-gelu epilogues, LayerNorm, causal attention), against the
unmodified transformers modules in fp32 - the oracle here IS the library the reference calls.  Random-init towers with
the SDXL head width (64): a quick-gelu tower without projection and an erf-gelu tower with text_projection."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu
transformers = pytest.importorskip("transformers")


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


class ToyTokenizer:
    def __call__(self, text, padding=None, max_length=77, truncation=True, return_tensors="pt"):
        ids = [1] + [3 + (sum(map(ord, w)) % 90) for w in text.split()][: max_length - 2] + [99]   # EOS = largest id
        ids = ids + [0] * (max_length - len(ids))
        return types.SimpleNamespace(input_ids=torch.tensor([ids]))


def _towers():
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    torch.manual_seed(0)
    c1 = CLIPTextConfig(vocab_size=100, hidden_size=192, intermediate_size=768, num_hidden_layers=4, num_attention_heads=3,
                        max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=2)
    c2 = CLIPTextConfig(vocab_size=100, hidden_size=320, intermediate_size=1280, num_hidden_layers=5, num_attention_heads=5,
                        max_position_embeddings=77, hidden_act="gelu", projection_dim=256, eos_token_id=2)
    e1, e2 = CLIPTextModel(c1).eval(), CLIPTextModelWithProjection(c2).eval()
    for e in (e1, e2):   # fp16-representable weights: the comparison measures the kernels, not the weight rounding
        for p in e.parameters():
            p.data = p.data.half().float()
    return e1, e2


def test_clip_towers_on_the_kernels_match_transformers():
    from omg_b200.text import ClipPromptEncoder, PackedClipText
    e1, e2 = _towers()
    tok = ToyTokenizer()
    ids = torch.cat([tok("a man and a woman on the beach").input_ids, tok("close-up photo of a dog , 35mm film").input_ids])
    with torch.no_grad():
        r1 = e1(ids, output_hidden_states=True)
        r2 = e2(ids, output_hidden_states=True)
    h1, p1 = PackedClipText(e1, "cuda")(ids)
    h2, p2 = PackedClipText(e2, "cuda")(ids)
    assert p1 is None and p2.shape == (2, 256)
    errs = (rel(h1, r1.hidden_states[-2]), rel(h2, r2.hidden_states[-2]), rel(p2, r2.text_embeds))
    print("clip towers rel err: penultimate L", errs[0], "penultimate bigG-style", errs[1], "text_embeds", errs[2])
    assert max(errs) < 1e-3   # measured on H100: 6.0e-4 / 6.6e-4 / 7.7e-4
    # the prompt encoder the pipelines use routes through the kernels on CUDA and keeps encode_prompt's layout
    import copy
    enc = ClipPromptEncoder([tok, tok], [copy.deepcopy(e1), copy.deepcopy(e2)], device="cuda", dtype=torch.float16)
    assert enc.use_kernels
    emb, pooled = enc("a man and a woman on the beach")
    assert emb.shape == (77, 192 + 320) and pooled.shape == (256,)
    assert rel(emb, torch.cat([r1.hidden_states[-2][0], r2.hidden_states[-2][0]], -1)) < 1e-3
    assert rel(pooled, r2.text_embeds[0]) < 1e-3
