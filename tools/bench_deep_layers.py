"""Measure StyleGAN2 conv-layer decomposition at 64 x 64 (convs.6) and 128 x 128 (convs.8) on one GPU.

Random init 1234, Z space, c = 80, B = NB = 2000.  Per layer it reports, as one JSON line:
  * ``job_s``: one whole ``get_or_compute`` (N = --n, with the regression pass) and ``peak_hbm_gb``, torch's peak allocation in it;
  * ``group_ms``: one partial_fit group, split into ``synthesis_ms`` (2000 rows written into the engine's stacked matrix),
    ``gram_ms`` (centring + small-side Gram), ``solve_ms`` (fp64 eigensolve + U^T M) and ``commit_ms``, medians over --steps;
  * ``export_ms``: the engine's export, the NHWC -> NCHW permutation of components, mean and variance (as the
    driver's export does), and their copy to the host.
Device times come from CUDA events; the job time from a host clock around work that ends in a synchronise.

    python tools/bench_deep_layers.py [--layers convs.6 convs.8] [--steps 3] [--n 6000] [--out results/deep_layers.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the card's name still comes from torch
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def bench_layer(layer, n, steps, c=80, b=2000):
    from ganspace_b200 import _native
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model)
    res, ch = model._synthesis(model.synthesis_layer_names().index(layer) + 1).shapes[-1]
    d = res * res * ch
    rec = {"layer": layer, "d": d, "c": c, "B": b, "NB": b, "N": n}

    # one whole job, twice: the first run warms the modules and the repack cache
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=False,
                 estimator="ipca")
    jobs = []
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(2):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=f"{tmp}/{rep}", run_dir_root=f"{tmp}/{rep}"),
                           force_recompute=True)
            torch.cuda.synchronize()
            jobs.append(time.perf_counter() - t0)
            peak = torch.cuda.max_memory_allocated(dev)
    rec["job_s"] = [round(t, 3) for t in jobs]
    rec["peak_hbm_gb"] = round(peak / 1e9, 2)
    torch.cuda.empty_cache()

    # the phases of one group on the engine's own C ABI (what BigIPCA.step runs), the batch synthesised into its rows
    eng = _native.BigIPCA(d, c, b, dev)
    lib = _native.load()
    tail = lambda: (_native._ptr(eng.ws), eng.ws.numel(), _native._stream())
    args = lambda: (_native._ptr(eng.state), _native._ptr(eng.M), eng.d, eng.c, eng.nb_max, eng.n_seen, b, eng.flags)
    ph = {"synthesis_ms": [], "gram_ms": [], "solve_ms": [], "commit_ms": []}
    for s in range(steps + 1):                     # step 0 warms up (and is the first partial_fit, which has no S*Vt rows)
        z = model.sample_latent(b, seed=1000 + s)
        t_syn, _ = timed(lambda: model.activations_into(z, layer, eng.batch_rows(b)))
        t_gram, _ = timed(lambda: _native._check(lib.gsb_bigd_step_gram(*args(), _native._ptr(eng.batch_mean), *tail()), "gram"))
        t_solve, _ = timed(lambda: _native._check(lib.gsb_bigd_step_solve(*args(), None, *tail()), "solve"))
        t_commit, _ = timed(lambda: _native._check(lib.gsb_bigd_step_commit(*args(), None, *tail()), "commit"))
        eng.n_seen += b
        eng.last_nb = b
        if s > 0:
            for k, t in zip(ph, (t_syn, t_gram, t_solve, t_commit)):
                ph[k].append(t)
    for k, v in ph.items():
        rec[k] = round(median(v), 2)
    rec["group_ms"] = round(sum(rec[k] for k in ph), 2)

    def export():
        out = eng.export()
        return {k: (_native.nhwc_to_nchw_rows(out[k].reshape(-1, d), res * res, ch) if k in ("components", "mean", "var") else out[k])
                .cpu() for k in out}
    export()
    rec["export_ms"] = round(median([timed(export)[0] for _ in range(3)]), 1)
    rec["engine_gb"] = round(_native.BigIPCA.device_bytes(d, c, b) / 1e9, 2)
    del eng
    inst.close()
    torch.cuda.empty_cache()
    _native.scratch.clear()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", nargs="+", default=["convs.6", "convs.8"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--n", type=int, default=6000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deep_layers: no CUDA device (the measurement runs on the GPU only)")
    gpu = gpu_info()
    lines = []
    for layer in a.layers:
        rec = bench_layer(layer, a.n, a.steps)
        rec["gpu"] = gpu
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
