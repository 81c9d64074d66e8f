"""StyleGAN2 style space (ffhq 1024^2, random init 1234) on one GPU:

  * get_or_compute on convs.4.conv.modulation (W space, N = 10^6, B = 10^4, c = 80, estimator ipca), alternated with config 2's
    job (layer style, same N / B / c) on the same card;
  * StyleGAN2.forward at batch 1 and 8, without a hook and with an offset edit on convs.5.conv.modulation (CUDA events).
Prints one JSON line with the card's name, power limit and max SM clock, and writes it to --out.

    python tools/bench_stylespace.py [--reps 3] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _job(inst, layer, n, b, c):
    import torch
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=True, estimator="ipca")
    with tempfile.TemporaryDirectory() as tmp:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def _forward_ms(model, z, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    model.forward(z)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        model.forward(z)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ganspace_b200.models import StyleGAN2, get_instrumented_model
    if not torch.cuda.is_available():
        raise SystemExit("bench_stylespace needs a CUDA device")
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    res = {"gpu": _gpu_info(), "n": args.n, "batch": 10_000, "components": 80}
    jobs = {"convs.4.conv.modulation": [], "style": []}
    for layer in jobs:                                   # warm-up: packs, scratch buffers, module loads
        inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=True)
        _job(inst, layer, 100_000, 10_000, 80)
        inst.close()
    for _ in range(args.reps):
        for layer in jobs:
            inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=True)
            jobs[layer].append(_job(inst, layer, args.n, 10_000, 80))
            inst.close()
    res["get_or_compute_s"] = {k: v for k, v in jobs.items()}
    model.use_z()
    fwd = {}
    for bsz in (1, 8):
        z = model.sample_latent(bsz, seed=1)
        fwd[f"b{bsz}_plain_ms"] = _forward_ms(model, z, 10)
        inst = get_instrumented_model("StyleGAN2", "ffhq", "convs.5.conv.modulation", dev, model=model, use_w=False)
        inst.edit_layer("convs.5.conv.modulation", offset=torch.full((1, 512), 0.1, device=dev))
        fwd[f"b{bsz}_s_edit_ms"] = _forward_ms(model, z, 10)
        inst.close()
    res["forward"] = fwd
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
