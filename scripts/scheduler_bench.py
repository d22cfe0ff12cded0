"""Per-launch time of the denoising-step tail: omg_fuse_step (Euler on epsilon) and omg_solver_step for each rule of
omg_b200/scheduler.py, at a 128x128 latent (SDXL 1024^2) with 0 and 2 concepts, by CUDA events over many launches;
the algorithmic bytes per launch from the shapes; and the step tail's share of a config-2 call (SDXL, 1024^2, 30 steps,
two LoRA concepts) from the launch count of that call.  Prints the card name and power limit with the numbers, and
one JSON line."""
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from omg_b200 import ops  # noqa: E402
from omg_b200 import scheduler as S  # noqa: E402

BASE = S.SDXL_BASE_CONFIG
RULES = {
    "euler_v": S.EulerDiscreteScheduler.from_config(BASE, prediction_type="v_prediction"),
    "euler_a": S.cli_scheduler("euler_a", BASE),
    "dpmpp_2m": S.cli_scheduler("dpmpp_2m", BASE),
    "dpmpp_2m_sde": S.cli_scheduler("dpmpp_2m_sde", BASE),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def step_bytes(HW, n, history, noise):
    """Bytes the step must move: omg_fuse_step's (elementwise.cu header) plus history read + write and noise."""
    b = (4 + 2 * n) * HW * 8 * 2 + n * HW * 4 + HW * 2 * 4 * 4 + HW * 2 * 4 * 4 + 6 * HW * 8 * 2
    if history:
        b += 2 * HW * 2 * 4 * 4
    if noise:
        b += HW * 2 * 4 * 2
    return b


def time_launches(fn, iters=2000, warm=50):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def main():
    if not torch.cuda.is_available():
        raise SystemExit("scheduler_bench needs a CUDA device")
    dev = "cuda"
    h = w = 128
    HW = h * w
    print("card:", card())
    rows = []
    for n in (0, 2):
        nm = torch.randn(4, HW, 8, device=dev).half()
        ncs = [torch.randn(2, HW, 8, device=dev).half() for _ in range(n)]
        masks = [(torch.rand(HW, device=dev) < 0.4).float() for _ in range(n)]
        lat = torch.randn(2, h, w, 4, device=dev)
        nxt = torch.empty(4, h, w, 8, dtype=torch.float16, device=dev)
        nxc = torch.empty(2, h, w, 8, dtype=torch.float16, device=dev)
        hist = torch.zeros(2, h, w, 4, device=dev)
        z = torch.randn(2, 4, h, w, device=dev).half()
        cases = {"fuse_step (euler eps)": (lambda: ops.fuse_step(nm, ncs, masks, 7.5, 5.0, 4.2, lat, nxt, nxc), False, False)}
        for name, s in RULES.items():
            s.set_timesteps(30)
            k = s.step_coeffs(5)
            cases[f"solver_step {name}"] = (
                (lambda k=k, s=s: ops.solver_step(nm, ncs, masks, 7.5, k, lat, nxt, nxc, history=hist,
                                                  store_x0=s.uses_history, noise=z if k.d else None)),
                s.uses_history, k.d != 0)
        for name, (fn, hs, nz) in cases.items():
            us = time_launches(fn)
            b = step_bytes(HW, n, hs, nz)
            rows.append({"kernel": name, "concepts": n, "us": round(us, 2), "MB": round(b / 1e6, 2),
                         "GB/s": round(b / us / 1e3, 1)})
            print(f"{name:32s} n={n}  {us:7.2f} us  {b / 1e6:6.2f} MB  {b / us / 1e3:7.1f} GB/s")
    # the step tail in a config-2 call: 30 step launches; the call time comes from bench-sized runs of the pipeline
    from omg_b200 import factory
    wl = factory.build_lora_workload(None, 1024, 2, 32, 30, 7.5)
    kw = dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(14)).half()
    for _ in range(2):
        wl.pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw)
        wl.controller.reset()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    wl.pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw)
    e1.record()
    torch.cuda.synchronize()
    wl.controller.reset()
    call_ms = e0.elapsed_time(e1)
    tail = {r["kernel"]: r["us"] for r in rows if r["concepts"] == 2}
    # 16 steps without fusion (0 concepts) + 14 with it (2 concepts) would be config 2's mix; the 2-concept time bounds it
    share = {k: round(30 * v / 1e3 / call_ms, 6) for k, v in tail.items()}
    print(f"config-2 stage-2 call: {call_ms:.1f} ms; 30 step tails at the 2-concept time are a share of {share}")
    print(json.dumps({"card": card(), "rows": rows, "config2_stage2_call_ms": round(call_ms, 2), "tail_share": share}))


if __name__ == "__main__":
    main()
