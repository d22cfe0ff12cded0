"""Same-box A/B of library builds for the fp16 VAE decode: decodes seeded latents with synthetic SDXL-width weights
(2 images at 32 x 32 and 1 at 128 x 128 latents) under each build and reports whether the images are bit-identical.

    python scripts/vae_ab.py LIB_A LIB_B    # paths of two libomg_b200.so builds

Each build runs in its own process (OMG_B200_LIB=<path>); one JSON line with the SHA-256 of every image per build."""
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import hashlib, json, sys
import torch
sys.path.insert(0, ".")
from omg_b200 import synthetic
from omg_b200.vae import PackedVaeDecoder, VaeConfig
cfg = VaeConfig.sdxl()
dec = PackedVaeDecoder(synthetic.make_vae_state_dict(cfg, 0), cfg)
out = {}
for B, h, w, seed in ((2, 32, 32, 1), (1, 128, 128, 2)):
    lat = (torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(seed)) * 0.4).half().cuda()
    img = dec.decode(lat).contiguous()
    torch.cuda.synchronize()
    out[f"{B}x{h}x{w}"] = hashlib.sha256(img.view(torch.int16).cpu().numpy().tobytes()).hexdigest()
print(json.dumps(out))
"""


def run(lib):
    env = dict(os.environ, OMG_B200_LIB=os.path.abspath(lib))
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    a, b = run(sys.argv[1]), run(sys.argv[2])
    print(json.dumps({"name": "vae_decode_fp16_ab", "bit_identical": a == b, "a": a, "b": b,
                      "libs": [hashlib.sha256(open(p, "rb").read()).hexdigest()[:12] for p in sys.argv[1:]]}))


if __name__ == "__main__":
    main()
