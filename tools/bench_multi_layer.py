"""Every StyleGAN2 style layer (ffhq 1024^2, random init 1234, W space, N = 10^6, B = 10^4, c = 80, estimator ipca) on one GPU:
the per-layer loop (get_or_compute with force_recompute, one layer after another) alternated with one get_or_compute_layers
pass, --reps of each.  Checks that the two sets of files hold the same arrays byte for byte (every .npy member of every .npz;
the zip containers differ only in their timestamps).  Prints one JSON line with the card's name, power limit and max SM clock,
and writes it to --out.

    python tools/bench_multi_layer.py [--reps 3] [--n 1000000] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
import tempfile
import time
import zipfile
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


def _cfg(layer, n):
    from ganspace_b200.config import Config
    return Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=80, n=n, batch_size=10_000, use_w=True,
                  estimator="ipca")


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def _loop(model, layers, n, run_dir):
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    sub = SimpleNamespace(run_dir=run_dir, run_dir_root=run_dir)
    paths = {}
    for layer in layers:
        inst = get_instrumented_model("StyleGAN2", "ffhq", layer, model.device, model=model, use_w=True)
        paths[layer] = get_or_compute(_cfg(layer, n), inst, submit_config=sub, force_recompute=True)
        inst.close()
    return paths


def _joint(model, layers, n, run_dir):
    from ganspace_b200.decomposition import get_or_compute_layers
    from ganspace_b200.models import get_instrumented_model
    sub = SimpleNamespace(run_dir=run_dir, run_dir_root=run_dir)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layers, model.device, model=model, use_w=True)
    paths = get_or_compute_layers(_cfg(layers[0], n), layers, inst, submit_config=sub, force_recompute=True)
    inst.close()
    return paths


def _members(path):
    with zipfile.ZipFile(path) as z:
        return {name: z.read(name) for name in sorted(z.namelist())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ganspace_b200.models import StyleGAN2
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_layer needs a CUDA device")
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    layers = [t[0] for t in model.model.style_layers()]
    res = {"gpu": _gpu_info(), "n": args.n, "batch": 10_000, "components": 80, "layers": len(layers)}
    with tempfile.TemporaryDirectory() as tmp:
        loop_dir, joint_dir = str(Path(tmp) / "loop"), str(Path(tmp) / "joint")
        _loop(model, layers, 100_000, loop_dir)           # warm-up: packs, scratch buffers, chain streams
        _joint(model, layers, 100_000, joint_dir)
        loop_s, joint_s = [], []
        for _ in range(args.reps):
            t, loop_paths = _timed(lambda: _loop(model, layers, args.n, loop_dir))
            loop_s.append(t)
            t, joint_paths = _timed(lambda: _joint(model, layers, args.n, joint_dir))
            joint_s.append(t)
        same = all(loop_paths[l].name == joint_paths[l].name and _members(loop_paths[l]) == _members(joint_paths[l])
                   for l in layers)
    res.update({"per_layer_loop_s": loop_s, "joint_s": joint_s, "files_identical": same})
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")
    if not same:
        raise SystemExit("the joint pass's files differ from the per-layer files")


if __name__ == "__main__":
    main()
