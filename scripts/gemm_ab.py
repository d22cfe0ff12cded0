"""Per-shape GEMM timing of the SDXL UNet's Linear / conv shapes (main forward B = 4, grouped forward B = 8) for same-box
A/B of library builds.

  python scripts/gemm_ab.py                        time the library _lib.py loads (OMG_B200_LIB=<path> selects a build)
  python scripts/gemm_ab.py --libs A.so B.so [--rounds 3]
                                                   alternate the builds (A, B) x rounds, each run in its own process, and
                                                   print per shape the median and spread over rounds of every build

Every launch uses the automatic tile choice and the epilogue the UNet uses (GEGLU for ff1, a residual for attn-out / ff2);
each residual shape also runs as the transformer blocks run it - in place (out = residual) with row statistics out
(`_inplace`) - and with the same row statistics but no residual (`_plain`), so the residual's own cost is the gap
between those two rows.  A timed launch is the median of 20 CUDA-event-timed launches with L2 flushed before each.  One JSON line per shape."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (tag, M per image-batch of 4, N, K, kind): level 2 = 32 x 32 tokens, level 1 = 64 x 64 tokens per image at 1024^2
LINEARS = [("l2_ff1_geglu", 4096, 10240, 1280, "geglu"), ("l2_qkv", 4096, 3840, 1280, "plain"),
           ("l2_out", 4096, 1280, 1280, "residual"), ("l2_ff2", 4096, 1280, 5120, "residual"),
           ("l1_ff1_geglu", 16384, 5120, 640, "geglu"), ("l1_qkv", 16384, 1920, 640, "plain"),
           ("l1_out", 16384, 640, 640, "residual"), ("l1_ff2", 16384, 640, 2560, "residual")]
# (tag, H = W, Cin, N) 3x3 convs of the ResBlocks (B = 4 images)
CONVS = [("conv320@128", 128, 320, 320), ("conv960->320@128", 128, 960, 320), ("conv640@64", 64, 640, 640),
         ("conv1280->640@64", 64, 1280, 640), ("conv1280@32", 32, 1280, 1280), ("conv2560->1280@32", 32, 2560, 1280)]


def measure():
    import torch
    sys.path.insert(0, ROOT)
    from omg_b200 import _lib as L
    from omg_b200 import ops

    dev = "cuda"
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def timeit(fn, iters=20, warm=3):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, device=dev) * scale).half()

    rows = []
    for batch in (4, 8):
        for tag, M, N, K, kind in LINEARS:
            M = M * batch // 4
            x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
            res = rnd(M, N) if kind == "residual" else None
            out = torch.empty(M, N // 2 if kind == "geglu" else N, device=dev, dtype=torch.float16)
            epi = L.EPI_GEGLU if kind == "geglu" else L.EPI_NONE
            ms = timeit(lambda: ops.linear(x, w, residual=res, out=out, epilogue=epi))
            row = {"M": M, "N": N, "K": K, "gflop": 2.0 * M * N * K / 1e9}
            rows.append({"name": f"{tag}_b{batch}", **row, "us": ms * 1e3})
            if kind == "residual":
                stats = torch.empty(ops.gemm_plan(N, L.EPI_NONE, M)[1], M, 2, device=dev)
                ms = timeit(lambda: ops.linear(x, w, residual=out, out=out, stats_out=stats))
                rows.append({"name": f"{tag}_inplace_b{batch}", **row, "us": ms * 1e3})
                ms = timeit(lambda: ops.linear(x, w, out=out, stats_out=stats))
                rows.append({"name": f"{tag}_plain_b{batch}", **row, "us": ms * 1e3})
                del stats
            del x, w, res, out
        for tag, H, Cin, N in CONVS:
            x = rnd(batch, H, H, Cin)
            w = ops.pack_conv3x3_weight(rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
            out = torch.empty(batch, H, H, N, device=dev, dtype=torch.float16)
            ms = timeit(lambda: ops.conv3x3(x, w, out=out))
            rows.append({"name": f"{tag}_b{batch}", "M": batch * H * H, "N": N, "K": 9 * Cin,
                         "gflop": 2.0 * batch * H * H * N * 9 * Cin / 1e9, "us": ms * 1e3})
            del x, w, out
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="*", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not args.libs:
        rows = measure()
        if args.child:
            print(json.dumps(rows))
            return
        for r in rows:
            r["tflops"] = round(r["gflop"] / r["us"] * 1e3, 1)
            r["us"] = round(r["us"], 1)
            print(json.dumps(r), flush=True)
        return
    runs = {lib: [] for lib in args.libs}
    for rnd_i in range(args.rounds):
        for lib in args.libs:
            env = dict(os.environ, OMG_B200_LIB=os.path.abspath(lib))
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True,
                               text=True, cwd=ROOT)
            if p.returncode != 0:
                sys.exit(f"{lib} round {rnd_i}: exit {p.returncode}\n{p.stderr[-4000:]}")
            runs[lib].append({r["name"]: r for r in json.loads(p.stdout.strip().splitlines()[-1])})
    for name, r0 in runs[args.libs[0]][0].items():
        out = {"name": name, "M": r0["M"], "N": r0["N"], "K": r0["K"], "gflop": round(r0["gflop"], 2)}
        for lib in args.libs:
            us = sorted(rr[name]["us"] for rr in runs[lib])
            med = us[len(us) // 2]
            out[os.path.basename(os.path.dirname(os.path.abspath(lib))) or lib] = {
                "us_median": round(med, 1), "us_spread": [round(us[0], 1), round(us[-1], 1)],
                "tflops": round(r0["gflop"] / med * 1e3, 1)}
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
