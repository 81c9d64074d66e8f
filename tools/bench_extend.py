"""get_or_extend from N1 to N2 samples against a fresh N2 get_or_compute, alternated in one process, --reps of each, at two
shapes (random init 1234, c = 80):
  * ``style``: StyleGAN2 ffhq W latents, B = 10^4, N = 10^6 -> 2 * 10^6;
  * ``convs4``: StyleGAN2 ffhq ``convs.4`` (32 x 32 x 512, the large-d engine), Z space with the regression pass, B = 2000,
    N = 20k -> 40k.
Each extension starts from the same saved state of the N1 run (copied back before every rep).  Also reported per shape: the
state's size and the times of its parts -- ``state_dict`` (device -> host), the file write, the file read and
``load_state_dict`` (host -> device) -- and whether the extended file's arrays equal the fresh run's.  Prints one JSON line
with the card's name, power limit and max SM clock, and writes it to --out.

    python tools/bench_extend.py [--reps 2] [--shapes style,convs4] [--scale 1.0] [--out FILE]
"""
import argparse
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = {
    # name: (layer, use_w, B, N1, N2)
    "style": ("style", True, 10_000, 1_000_000, 2_000_000),
    "convs4": ("convs.4", False, 2000, 20_000, 40_000),
}


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _cfg(layer, use_w, b, n):
    from ganspace_b200.config import Config
    return Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=80, n=n, batch_size=b, use_w=use_w,
                  estimator="ipca")


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


class _PartTimer:
    """Wall-clock of the state's save and load steps, by wrapping them."""

    def __init__(self):
        from ganspace_b200 import decomposition, estimators
        self.t = {}
        self._wrap(estimators.IPCAEstimator, "state_dict", "state_dict_s")
        self._wrap(estimators.IPCAEstimator, "load_state_dict", "load_state_dict_s")
        self._wrap(decomposition.StateFile, "load", "file_read_s")
        real_write = decomposition.StateFile.write.__func__
        timer = self

        def write(cls, *a, **k):
            t0 = time.perf_counter()
            out = real_write(cls, *a, **k)
            timer.t.setdefault("file_write_s", []).append(time.perf_counter() - t0)
            return out
        decomposition.StateFile.write = classmethod(write)

    def _wrap(self, owner, name, label):
        import torch
        real = getattr(owner, name)
        timer = self

        def fn(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = real(*a, **k)
            torch.cuda.synchronize()
            timer.t.setdefault(label, []).append(time.perf_counter() - t0)
            return out
        setattr(owner, name, fn)


def _arrays(path):
    import numpy as np
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def bench_shape(model, name, reps, scale, timer):
    import numpy as np
    from ganspace_b200.decomposition import _dump_path, _state_path, get_or_compute, get_or_extend
    from ganspace_b200.models import get_instrumented_model
    layer, use_w, b, n1, n2 = SHAPES[name]
    n1, n2 = (max(int(n * scale) // b * b, 2 * max(b, 2000)) for n in (n1, n2))
    n2 = max(n2, 2 * n1)
    model.use_w() if use_w else model.use_z()
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, model.device, model=model)
    res = {"layer": layer, "use_w": use_w, "batch": b, "n1": n1, "n2": n2, "components": 80}
    with tempfile.TemporaryDirectory() as tmp:
        fresh_sub = SimpleNamespace(run_dir=str(Path(tmp) / "fresh"), run_dir_root=tmp)
        ext_sub = SimpleNamespace(run_dir=str(Path(tmp) / "ext"), run_dir_root=tmp)
        c1, c2 = _cfg(layer, use_w, b, n1), _cfg(layer, use_w, b, n2)
        get_or_compute(_cfg(layer, use_w, b, 4 * max(2000, b)), inst, submit_config=fresh_sub, force_recompute=True)   # warm-up
        timer.t.clear()
        t_n1, _ = _timed(lambda: get_or_extend(c1, inst, submit_config=ext_sub))
        state = _state_path(_dump_path(ext_sub.run_dir, c1), c1)
        saved = Path(tmp) / "saved.gsbstate"
        shutil.copyfile(state, saved)
        res.update(n1_run_s=t_n1, state_bytes=saved.stat().st_size, state_dict_s=timer.t.get("state_dict_s"),
                   file_write_s=timer.t.get("file_write_s"))
        fresh_s, ext_s, reads, loads = [], [], [], []
        for _ in range(reps):
            t, fresh = _timed(lambda: get_or_compute(c2, inst, submit_config=fresh_sub, force_recompute=True))
            fresh_s.append(t)
            out = _dump_path(ext_sub.run_dir, c2)
            out.unlink(missing_ok=True)
            shutil.copyfile(saved, state)
            timer.t.clear()
            t, ext = _timed(lambda: get_or_extend(c2, inst, submit_config=ext_sub))
            ext_s.append(t)
            reads += timer.t.get("file_read_s", [])
            loads += timer.t.get("load_state_dict_s", [])
        a, e = _arrays(fresh), _arrays(ext)
        same = sorted(a) == sorted(e) and all(np.array_equal(a[k], e[k]) for k in a)
    inst.close()
    res.update(fresh_n2_s=fresh_s, extend_n1_to_n2_s=ext_s, file_read_s=reads, load_state_dict_s=loads, arrays_equal=same)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--shapes", default="style,convs4")
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies N1 and N2 (quick runs)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ganspace_b200.models import StyleGAN2
    if not torch.cuda.is_available():
        raise SystemExit("bench_extend needs a CUDA device")
    model = StyleGAN2(torch.device("cuda:0"), "ffhq", random_init=1234)
    timer = _PartTimer()
    res = {"gpu": _gpu_info(), "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        res["shapes"][name] = bench_shape(model, name, args.reps, args.scale, timer)
        print(json.dumps({name: res["shapes"][name]}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")
    if not all(r["arrays_equal"] for r in res["shapes"].values()):
        raise SystemExit("an extended file differs from the fresh run's")


if __name__ == "__main__":
    main()
