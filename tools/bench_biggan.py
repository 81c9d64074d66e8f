"""BigGAN-deep-512 (random init + synthesis_fill, husky) on one GPU: BigGAN.forward images/s at batch 1, 8 and 32, the per-module
CUDA-event split (generator.layers.k and the RGB tail) and the achieved TFLOP/s against the ~76 GFLOP of useful work per 512^2
image (the convs of every GenBlock, the SelfAttn products and the 3 kept channels of conv_to_rgb).  The batch sizes alternate,
rep by rep.  Prints one JSON line and writes it to --out.

    python tools/bench_biggan.py [--batches 1,8,32] [--steps 5] [--warmup 1] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def useful_gflop(model):
    """Multiply-adds x 2 of one image: the four convs of every GenBlock at their resolutions, the SelfAttn GEMMs (theta|phi|g,
    scores, weighted sum, o_conv) and conv_to_rgb restricted to the 3 channels the image keeps."""
    g = model.model.generator
    res, flop = 4, 0.0
    for layer in g.layers:
        if type(layer).__name__ == "SelfAttn":
            c, hw = layer.in_channels, res * res
            flop += hw * c * (c // 8 * 2 + c // 2) + hw * (hw // 4) * (c // 8) + hw * (hw // 4) * (c // 2) + hw * (c // 2) * c
            continue
        cin, mid, cout = layer.conv_0.weight_orig.shape[1], layer.conv_0.weight_orig.shape[0], layer.conv_3.weight_orig.shape[0]
        r2 = 2 * res if layer.up_sample else res
        flop += res * res * cin * mid + 2 * r2 * r2 * 9 * mid * mid + r2 * r2 * mid * cout
        res = r2
    flop += res * res * 9 * g.conv_to_rgb.weight_orig.shape[1] * 3
    return 2 * flop / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from ganspace_b200 import _native
    from ganspace_b200.models.biggan import BigGAN
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = BigGAN(dev, 512, "husky", random_init=4321)
    batches = [int(b) for b in args.batches.split(",")]
    gflop = useful_gflop(model)
    zs = {b: model.sample_latent(b, seed=100 + b) for b in batches}
    with torch.no_grad():
        for _ in range(args.warmup):
            for b in batches:
                model.forward(zs[b])
        torch.cuda.synchronize()
        times = {b: [] for b in batches}
        for _ in range(args.steps):
            for b in batches:                                      # alternated: each rep runs every batch size once
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                model.forward(zs[b])
                e1.record()
                torch.cuda.synchronize()
                times[b].append(e0.elapsed_time(e1))
        # per-module split at the largest batch (CUDA events around each module's launches)
        bmax = max(batches)
        _native.instrument.timing = True
        _native.instrument.reset()
        model.forward(zs[bmax])
        sections = _native.instrument.section_ms()
        _native.instrument.timing = False
    res = {"gpu": _gpu_info(), "useful_gflop_per_image": round(gflop, 2), "forward": {}}
    for b in batches:
        ms = sorted(times[b])[len(times[b]) // 2]
        res["forward"][str(b)] = {"median_ms": round(ms, 3), "min_ms": round(min(times[b]), 3), "max_ms": round(max(times[b]), 3),
                                  "images_per_s": round(1e3 * b / ms, 2), "ms_per_image": round(ms / b, 3),
                                  "tflops": round(gflop * b / ms, 2)}
    total = sum(v[0] for v in sections.values())
    res[f"modules_ms_batch{bmax}"] = {k: round(v[0], 3) for k, v in sorted(sections.items(), key=lambda kv: -kv[1][0])}
    res[f"modules_total_ms_batch{bmax}"] = round(total, 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
