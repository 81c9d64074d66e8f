"""ProGAN (random init, bedroom) on one GPU: get_or_compute at layer4 and layer10 (samples/s and the section split from CUDA
events: RNG, chain, IPCA step, regression, ...), ProGAN.forward at batch 5 and 64 (images/s), and the chain alone per block
(cumulative CUDA-event time of blocks 1..k at --chain-batch samples, differenced).  The jobs of the two layers alternate.
Prints one JSON line and writes it to --out.

    python tools/bench_progan.py [--n 20000] [--batch 500] [--components 80] [--steps 3] [--out FILE]
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


def _event_ms(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000)
    ap.add_argument("--batch", type=int, default=500)
    ap.add_argument("--components", type=int, default=80)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chain-batch", dest="chain_batch", type=int, default=64)
    ap.add_argument("--layers", default="layer4,layer10")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from ganspace_b200 import _native, decomposition
    from ganspace_b200.config import Config
    from ganspace_b200.models import ProGAN, get_instrumented_model
    dev = torch.device("cuda:0")
    model = ProGAN(dev, "bedroom", random_init=1234)
    layers = args.layers.split(",")
    insts = {}

    def job(layer, tmp):
        if layer not in insts:
            insts[layer] = get_instrumented_model("ProGAN", "bedroom", layer, dev, model=model)
        cfg = Config(model="ProGAN", layer=layer, output_class="bedroom", components=args.components, n=args.n,
                     batch_size=args.batch, estimator="ipca")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        decomposition.get_or_compute(cfg, insts[layer], submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    times, sections = {l: [] for l in layers}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.warmup):
            for l in layers:
                job(l, tmp)
        for _ in range(args.steps):
            for l in layers:
                times[l].append(job(l, tmp))
        for l in layers:                                     # section split in a run of its own (event pairs around every C call)
            _native.instrument.reset()
            _native.instrument.timing = True
            job(l, tmp)
            sections[l] = {k: round(v[0], 2) for k, v in _native.instrument.section_ms().items()}
            _native.instrument.timing = False
    for inst in insts.values():
        inst.close()

    images = {}
    for b in (5, 64):
        z = model.sample_latent(b, seed=1)
        ms = _event_ms(lambda: model.forward(z), 10)
        images[str(b)] = {"ms": round(ms, 3), "images_per_s": round(b / ms * 1e3, 1)}

    # the chain alone: blocks 1..k, differenced; GEMM FLOPs of block k = 2 * rows * cin * taps * cout * 3 (hi/lo split products)
    packed = model.model.packed()
    nb = args.chain_batch
    z = model.sample_latent(nb, seed=2).reshape(nb, -1)
    names = model.model.block_names()
    cum, per_block = 0.0, {}
    for k in range(1, packed.n_blocks + 1):
        ms = _event_ms(lambda: packed.forward(z, k), 5)
        d = packed.desc[k - 1]
        mma_flops = 2.0 * nb * d.res_in * d.res_in * d.cin * d.ksize * d.ksize * d.cout * 3
        step = max(ms - cum, 1e-6)
        per_block[names[k - 1]] = {"ms": round(ms - cum, 4), "mma_tflops": round(mma_flops / step / 1e9, 1)}
        cum = ms
    res = {
        "shape": f"ProGAN bedroom random-init N={args.n} B={args.batch} c={args.components}, one GPU",
        "gpu": _gpu_info(),
        "seconds_per_job": {l: [round(t, 3) for t in v] for l, v in times.items()},
        "samples_per_s_median": {l: round(args.n / sorted(v)[len(v) // 2], 1) for l, v in times.items()},
        "section_ms": sections,
        "forward": images,
        "chain_per_block": {"batch": nb, "blocks": per_block, "all_blocks_ms": round(cum, 3)},
    }
    model.check_numerics()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
