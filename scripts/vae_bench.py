"""VAE decode timing at the bench workload's size: 2 images, 128x128 latents -> 1024x1024, SDXL widths, synthetic
weights.  Prints one JSON line per storage type (ms per 2-image decode, algorithmic TFLOP/s, peak memory, the card's
name and power limit).

    python scripts/vae_bench.py [--dtype fp16,bf16] [--windows 9]

With several types the timed windows alternate between them in one process, on the same latents, so drift of the
clocks or of other work on the host hits each type alike; a last line gives the rel-L2 between their images."""
import argparse
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from omg_b200 import synthetic  # noqa: E402
from omg_b200.vae import PackedVaeDecoder, VaeConfig, vae_decoder_flops  # noqa: E402

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, watts = [x.strip() for x in r.stdout.strip().split(",")]
        return name, float(watts)
    except Exception:
        return torch.cuda.get_device_name(0), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="fp16", help="comma-separated storage types: fp16, bf16")
    ap.add_argument("--windows", type=int, default=5, help="timed decodes per type (median reported)")
    args = ap.parse_args()
    names = args.dtype.split(",")
    for n in names:
        if n not in DTYPES:
            raise SystemExit(f"--dtype {n}: expected one of {sorted(DTYPES)}")
    cfg = VaeConfig.sdxl()
    sd = synthetic.make_vae_state_dict(cfg, 0)
    decs = {n: PackedVaeDecoder(sd, cfg, dtype=DTYPES[n]) for n in names}
    B, h, w = 2, 128, 128
    lat = (torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(0)) * 0.4).half().cuda()
    imgs, peak = {}, {}
    for n in names:  # warm-up (module load, first launches) and each type's peak memory on its own
        for _ in range(2):
            imgs[n] = decs[n].decode(lat)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        imgs[n] = decs[n].decode(lat)
        torch.cuda.synchronize()
        peak[n] = torch.cuda.max_memory_allocated()
        imgs[n] = imgs[n].float()
    ts = {n: [] for n in names}
    for _ in range(args.windows):
        for n in names:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            decs[n].decode(lat)
            e1.record()
            torch.cuda.synchronize()
            ts[n].append(e0.elapsed_time(e1))
    gpu, watts = card()
    fl = B * vae_decoder_flops(cfg, h, w)
    for n in names:
        t = sorted(ts[n])
        ms = t[len(t) // 2]
        print(json.dumps({"name": "vae_decode_2x1024", "dtype": n, "ms": round(ms, 3), "ms_min": round(t[0], 3),
                          "ms_max": round(t[-1], 3), "tflops": round(fl / ms / 1e9, 1),
                          "algorithmic_tflop": round(fl / 1e12, 2), "finite": bool(torch.isfinite(imgs[n]).all()),
                          "peak_mem_gb": round(peak[n] / 2 ** 30, 2), "gpu": gpu, "power_limit_w": watts}))
    if len(names) > 1:
        a, b = imgs[names[0]], imgs[names[1]]
        print(json.dumps({"name": "vae_decode_2x1024_rel_l2", "pair": f"{names[1]}_vs_{names[0]}",
                          "rel_l2": float((b - a).norm() / a.norm())}))


if __name__ == "__main__":
    main()
