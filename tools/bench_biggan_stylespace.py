"""BigGAN-deep conditional-BatchNorm row layers (BigGAN-512 husky, random init 4321) on one GPU:

  * get_or_compute on a wide row layer (generator.layers.0.bn_0.scale, C = 2048; Z space, N = 10^6, B = 10^4, c = 80, ipca),
    alternated in one process with the generator.gen_z job of the same N / B / c (both on the exact low-rank path);
  * BigGAN.forward at batch 1, 8 and 32: plain, with retain hooks on the eight row layers of generator.layers.3, and with an
    offset edit on generator.layers.3.bn_2.scale; the three variants alternated, CUDA-event time per call.
Prints one JSON line with the card's name, power limit and max SM clock, and writes it to --out.

    python tools/bench_biggan_stylespace.py [--reps 3] [--n 1000000] [--out FILE]
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
ROW_LAYER = "generator.layers.0.bn_0.scale"
BLOCK = 3
EDIT_LAYER = f"generator.layers.{BLOCK}.bn_2.scale"


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _job(m, layer, n, reps_out):
    import torch
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    inst = get_instrumented_model("BigGAN-512", "husky", layer, torch.device("cuda:0"), model=m)
    cfg = Config(model="BigGAN-512", layer=layer, output_class="husky", components=80, n=n, batch_size=10_000)
    try:
        with tempfile.TemporaryDirectory() as tmp:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
            torch.cuda.synchronize()
            reps_out.append(time.perf_counter() - t0)
    finally:
        inst.close()


def _forward_ms(m, z, calls):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        m.forward(z)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import contextlib
    import io
    import torch
    from ganspace_b200.models.biggan import BigGAN
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    dev = torch.device("cuda:0")
    m = BigGAN(dev, 512, "husky", random_init=4321)
    res = {"gpu": _gpu_info(), "n": a.n, "batch_size": 10_000, "components": 80}

    times = {"row": [], "gen_z": []}
    for r in range(a.reps + 1):                          # the first round warms up (packing, QR, allocator)
        for key, layer in (("row", ROW_LAYER), ("gen_z", "generator.gen_z")):
            out = [] if r == 0 else times[key]
            with contextlib.redirect_stdout(io.StringIO()):
                _job(m, layer, a.n, out)
    res["row_job_s"] = times["row"]
    res["gen_z_job_s"] = times["gen_z"]

    rows = [f"generator.layers.{BLOCK}.bn_{j}.{kind}" for j in range(4) for kind in ("scale", "offset")]
    for bsz in (1, 8, 32):
        z = m.sample_latent(bsz, seed=1)
        variants = {}

        def plain():
            return None

        def retain():
            inst = InstrumentedModel(m)
            inst.retain_layers(rows)
            return inst

        def edit():
            inst = InstrumentedModel(m)
            inst.edit_layer(EDIT_LAYER, offset=torch.full((1, 512), 0.5, device=dev))
            return inst
        for name, setup in (("plain", plain), ("retain", retain), ("edit", edit)):
            inst = setup()
            m.forward(z)
            torch.cuda.synchronize()
            if inst is not None:
                inst.close()
        for _ in range(a.reps):
            for name, setup in (("plain", plain), ("retain", retain), ("edit", edit)):
                inst = setup()
                variants.setdefault(name, []).append(round(_forward_ms(m, z, a.calls), 3))
                if inst is not None:
                    inst.close()
        for name, v in variants.items():
            res[f"forward_b{bsz}_{name}_ms"] = v
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
