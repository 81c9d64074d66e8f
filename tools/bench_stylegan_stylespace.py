"""StyleGAN (v1) style space (ffhq 1024^2, random init 1234) on one GPU:

  * the style GEMM alone (gsb_stylegan_styles) at 10^6 rows x 1024 columns (g_synthesis.blocks.32x32.epi2.style_mod.lin):
    CUDA-event time per launch and the achieved FP32 rate against the H100 SXM data sheet's 67 TFLOP/s;
  * get_or_compute on g_synthesis.blocks.32x32.epi2.style_mod.lin (W space, N = 10^6, B = 10^4, c = 80, estimator ipca),
    alternated with the g_mapping job of the same N / B / c on the same card;
  * StyleGAN.forward at batch 1 and 8, without a hook and with an offset edit on g_synthesis.blocks.16x16.epi2.style_mod.lin
    (CUDA events).  With --parent DIR (another checkout of this package, built), the plain forward is also timed there, in
    subprocesses alternated with this tree's.
Prints one JSON line with the card's name, power limit and max SM clock, and writes it to --out.

    python tools/bench_stylegan_stylespace.py [--reps 3] [--n 1000000] [--parent DIR] [--out FILE]
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
STYLE_LAYER = "g_synthesis.blocks.32x32.epi2.style_mod.lin"
EDIT_LAYER = "g_synthesis.blocks.16x16.epi2.style_mod.lin"
FP32_PEAK = 67e12                  # H100 SXM data sheet, dense FP32, at up to 700 W

# StyleGAN.forward at batch 1 and 8 (no hook), ms per call; run with the working directory at the checkout to time
FORWARD_CHILD = r'''
import json, sys
import torch
sys.path.insert(0, ".")
from ganspace_b200.models import StyleGAN
dev = torch.device("cuda:0")
m = StyleGAN(dev, "ffhq", random_init=1234)
out = {}
for bsz in (1, 8):
    z = m.sample_latent(bsz, seed=1)
    for _ in range(3):
        m.forward(z)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        m.forward(z)
    e1.record()
    torch.cuda.synchronize()
    out[f"b{bsz}_plain_ms"] = e0.elapsed_time(e1) / REPS
print("RESULT " + json.dumps(out))
'''


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
    cfg = Config(model="StyleGAN", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=True, estimator="ipca")
    with tempfile.TemporaryDirectory() as tmp:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def _events_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _forward_in(tree, reps):
    r = subprocess.run([sys.executable, "-c", FORWARD_CHILD.replace("REPS", str(reps))], cwd=tree, capture_output=True, text=True)
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    if not line:
        raise SystemExit(f"forward timing in {tree} failed:\n{r.stderr[-2000:]}")
    return json.loads(line[0][len("RESULT "):])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--parent", default=None, help="a built checkout to time StyleGAN.forward against")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ganspace_b200.models import StyleGAN, get_instrumented_model
    if not torch.cuda.is_available():
        raise SystemExit("bench_stylegan_stylespace needs a CUDA device")
    dev = torch.device("cuda:0")
    model = StyleGAN(dev, "ffhq", random_init=1234)
    res = {"gpu": _gpu_info(), "n": args.n, "batch": 10_000, "components": 80}

    # the style GEMM alone
    packed = model.model.g_synthesis.packed()
    layer = [t[1] for t in model.model.style_layers() if t[0] == STYLE_LAYER][0]
    w = torch.randn((1, args.n, 512), device=dev)
    ms = _events_ms(lambda: packed.styles(w, [layer]), 10)
    flop = 2.0 * args.n * packed.style_width(layer) * 512
    res["style_gemm"] = {"rows": args.n, "cols": packed.style_width(layer), "ms": ms, "tflops": flop / ms / 1e9,
                         "share_of_67_tflops": flop / ms / 1e-3 / FP32_PEAK}
    del w
    torch.cuda.empty_cache()

    jobs = {STYLE_LAYER: [], "g_mapping": []}
    for layer_name in jobs:                                   # warm-up: packs, scratch buffers, module loads
        inst = get_instrumented_model("StyleGAN", "ffhq", layer_name, dev, model=model, use_w=True)
        _job(inst, layer_name, 100_000, 10_000, 80)
        inst.close()
    for _ in range(args.reps):
        for layer_name in jobs:
            inst = get_instrumented_model("StyleGAN", "ffhq", layer_name, dev, model=model, use_w=True)
            jobs[layer_name].append(_job(inst, layer_name, args.n, 10_000, 80))
            inst.close()
    res["get_or_compute_s"] = jobs
    model.use_z()

    fwd = {}
    for bsz in (1, 8):
        z = model.sample_latent(bsz, seed=1)
        fwd[f"b{bsz}_plain_ms"] = _events_ms(lambda: model.forward(z), 20)
        inst = get_instrumented_model("StyleGAN", "ffhq", EDIT_LAYER, dev, model=model, use_w=False)
        inst.edit_layer(EDIT_LAYER, offset=torch.full((1, 1024), 0.1, device=dev))
        fwd[f"b{bsz}_s_edit_ms"] = _events_ms(lambda: model.forward(z), 20)
        inst.close()
    res["forward"] = fwd
    if args.parent:
        runs = {"this": [], "parent": []}
        for _ in range(args.reps):
            runs["this"].append(_forward_in(ROOT, 20))
            runs["parent"].append(_forward_in(Path(args.parent).resolve(), 20))
        res["forward_alternated"] = runs
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
