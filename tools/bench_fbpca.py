"""--est fbpca at the config-2 shape (StyleGAN2-ffhq random-init, layer=style --use_w, N = 1e6, B = 10k, c = 80):
ms per get_or_compute job, alternated with --est ipca in the same process, and fbpca's phase split from CUDA events
(production = latent RNG + mapping + batch statistics; pooling = Chan folds of the group statistics; solve = range finder +
eigensolve + stdevs).  Prints one JSON line and writes it to --out.

    python tools/bench_fbpca.py [--steps 5] [--n 1000000]          (GPU)
    python tools/bench_fbpca.py --reference-cpu [--ref-n 40000]     (CPU: the unmodified reference with the restated fbpca
                                                                     installed as its fbpca module, bounded N, labelled so)
    python tools/bench_fbpca.py --config4 [--steps 5]               (GPU: config 4's layer, BigGAN-512 husky random-init
                                                                     generator.gen_z, N = 1e6, B = 1e4: fbpca at c = 16 and
                                                                     c = 80, each alternated with ipca at the same c, and the
                                                                     host draw of fbpca's [32768, 32] test matrix alone)
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


def run_gpu(args):
    import torch
    from ganspace_b200 import _native, decomposition
    from ganspace_b200.config import Config
    from ganspace_b200.models import StyleGAN2, get_instrumented_model
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", "style", dev, model=model, use_w=True)

    def job(est, tmp):
        cfg = Config(model="StyleGAN2", layer="style", output_class="ffhq", components=args.components, n=args.n,
                     batch_size=args.batch, use_w=True, estimator=est)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        decomposition.get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp),
                                     force_recompute=True)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    times = {"fbpca": [], "ipca": []}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.warmup):
            for est in times:
                job(est, tmp)
        for _ in range(args.steps):
            for est in times:
                times[est].append(job(est, tmp))
        _native.instrument.reset()
        _native.instrument.timing = True
        job("fbpca", tmp)
        sections = {k: round(v[0], 3) for k, v in _native.instrument.section_ms().items()}
        _native.instrument.timing = False
    production = sum(v for k, v in sections.items() if k not in ("fbpca_pool", "fbpca_solve"))
    res = {
        "shape": f"StyleGAN2-ffhq random-init style --use_w N={args.n} B={args.batch} c={args.components}",
        "gpu": _gpu_info(),
        "ms_per_job": {k: [round(t, 1) for t in v] for k, v in times.items()},
        "ms_per_job_median": {k: round(sorted(v)[len(v) // 2], 1) for k, v in times.items()},
        "fbpca_phase_ms": {"production": round(production, 3), "pooling": sections.get("fbpca_pool"),
                           "solve": sections.get("fbpca_solve"), "sections": sections},
    }
    return res


def run_config4(args):
    """gen_z: l = 32 < rank takes the randomized branch (host draw of Omega + projection), l = 160 the exact one."""
    import numpy as np
    import torch
    from ganspace_b200 import decomposition
    from ganspace_b200.config import Config
    from ganspace_b200.models import get_instrumented_model
    from ganspace_b200.models.biggan import BigGAN
    dev = torch.device("cuda:0")
    model = BigGAN(dev, 512, "husky", random_init=4321)
    inst = get_instrumented_model("BigGAN-512", "husky", "generator.gen_z", dev, model=model)

    def job(est, c, tmp):
        cfg = Config(model="BigGAN-512", layer="generator.gen_z", output_class="husky", components=c, n=args.n,
                     batch_size=args.batch, estimator=est)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        decomposition.get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp),
                                     force_recompute=True)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    jobs = [("fbpca", 16), ("ipca", 16), ("fbpca", 80), ("ipca", 80)]
    times = {f"{e}_c{c}": [] for e, c in jobs}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.warmup):
            for e, c in jobs:
                job(e, c, tmp)
        for _ in range(args.steps):
            for e, c in jobs:
                times[f"{e}_c{c}"].append(job(e, c, tmp))
    draw = []
    for _ in range(5):
        t0 = time.perf_counter()
        np.random.uniform(low=-1.0, high=1.0, size=(32768, 32)).astype(np.float32)
        draw.append((time.perf_counter() - t0) * 1e3)
    return {
        "shape": f"BigGAN-512 husky random-init generator.gen_z N={args.n} B={args.batch}",
        "gpu": _gpu_info(),
        "ms_per_job": {k: [round(t, 1) for t in v] for k, v in times.items()},
        "ms_per_job_median": {k: round(sorted(v)[len(v) // 2], 1) for k, v in times.items()},
        "host_omega_draw_ms_c16": [round(t, 2) for t in draw],
    }


def run_profile(args):
    """Kernel table of the solve alone (torch.profiler, CUDA activities) on a synthetic pooled state of the bench's shape."""
    import numpy as np
    import torch
    from ganspace_b200 import _native
    dev = torch.device("cuda:0")
    d, c = 512, args.components
    rng = np.random.RandomState(0)
    X = torch.from_numpy((rng.standard_normal((20_000, d)) * (0.99 ** np.arange(d))[None, :]).astype(np.float32)).to(dev)
    mean, gram = _native.batch_stats(X)
    pool = _native.FBPCAPool(d, dev)
    pool.accumulate(20_000, mean.reshape(1, d), gram.reshape(1, d, d))
    omega = torch.from_numpy(rng.uniform(-1, 1, (d, 2 * c))).to(dev)
    for _ in range(3):
        pool.solve(c, 2 * c, omega=omega)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            pool.solve(c, 2 * c, omega=omega)
        torch.cuda.synchronize()
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
    return {"gpu": _gpu_info(), "profile_5_solves": table}


def run_reference_cpu(args):
    import numpy as np
    import torch
    from oracle import fbpca_oracle, ref_harness
    sys.modules["fbpca"] = fbpca_oracle
    ref = ref_harness.import_reference()
    m = ref_harness.rand_init_stylegan2(ref, torch.device("cpu"), "ffhq")
    inst = ref.wrappers.get_instrumented_model("StyleGAN2", "ffhq", "style", torch.device("cpu"), model=m, use_w=True)
    cfg = ref.Config(model="StyleGAN2", layer="style", output_class="ffhq", estimator="fbpca", use_w=True, n=args.ref_n,
                     batch_size=args.batch, components=args.components)
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        ref.decomposition.get_or_compute(cfg, inst, force_recompute=True,
                                         submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
        dt = time.perf_counter() - t0
    return {"label": "unmodified reference on the host CPU with the restated fbpca (oracle/fbpca_oracle.py) as its fbpca "
                     f"module, bounded N={args.ref_n}", "threads": torch.get_num_threads(), "seconds": round(dt, 2),
            "numpy": np.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--components", type=int, default=80)
    ap.add_argument("--reference-cpu", dest="reference_cpu", action="store_true")
    ap.add_argument("--ref-n", dest="ref_n", type=int, default=40_000)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--config4", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.profile:
        res = run_profile(args)
        print(res["profile_5_solves"])
    elif args.config4:
        res = run_config4(args)
    else:
        res = run_reference_cpu(args) if args.reference_cpu else run_gpu(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
