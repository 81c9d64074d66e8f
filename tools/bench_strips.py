"""Frames/s of component strips, the reference's loop against ganspace_b200.strips, alternated in one process, --reps of each:
  * ``first_20_pcs``: StyleGAN2 ffhq (1024^2) in W, 20 components x 7 frames x 1 latent, centred (figure_first_20_pcs);
  * ``visualize``: StyleGAN (v1) ffhq (1024^2) in W, 10 components x 5 frames x 5 latents, centred (visualize.py's grids).
The reference path is tests/strip_reference.py: one call per component, five frames per ``sample_np``, latents built with torch
ops per call.  The new path is one ``create_strip_centered(..., per_component=True)`` call.  Both end with every frame as a
float32 NumPy array on the host.  Random init 1234.  Prints one JSON line per workload (medians and every rep) with the card's
name, power limit and max SM clock.

Activation edits (``mode='activation'``; the reference loop over ``inst.edit_layer``, tests/act_strip_reference.py):
  * ``act_style_z``: StyleGAN2 ffhq in Z, ``style``, 14 components x 5 frames x 1 latent, centred (visualize.py's summary grid);
  * ``act_modulation_w``: StyleGAN2 ffhq in W, ``convs.4.conv.modulation``, 20 components x 7 frames x 1 latent;
  * ``act_gen_z``: BigGAN-512 husky, ``generator.gen_z``, 14 components x 5 frames x 1 latent, centred.

    python tools/bench_strips.py [--reps 3] [--workloads first_20_pcs,visualize,act_style_z,act_modulation_w,act_gen_z]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

WORKLOADS = {
    # name: (model, class, n_comp, n_frames, n_lat)
    "first_20_pcs": ("StyleGAN2", "ffhq", 20, 7, 1),
    "visualize": ("StyleGAN", "ffhq", 10, 5, 5),
}
ACT_WORKLOADS = {
    # name: (model, class, layer, space, n_comp, n_frames, n_lat, centred)
    "act_style_z": ("StyleGAN2", "ffhq", "style", "Z", 14, 5, 1, True),
    "act_modulation_w": ("StyleGAN2", "ffhq", "convs.4.conv.modulation", "W", 20, 7, 1, False),
    "act_gen_z": ("BigGAN-512", "husky", "generator.gen_z", "Z", 14, 5, 1, True),
}


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _inst(name, cls, dev):
    from ganspace_b200.models import StyleGAN, StyleGAN2, get_instrumented_model, stylegan
    if name == "StyleGAN2":
        return get_instrumented_model(name, cls, "style", dev, model=StyleGAN2(dev, cls, random_init=1234), use_w=True)
    m = StyleGAN(dev, cls, random_init=1234)
    stylegan.synthesis_fill(m.model, 7)
    return get_instrumented_model(name, cls, "g_mapping", dev, model=m, use_w=True)


def _act_inst(name, cls, space, dev):
    from ganspace_b200.models import StyleGAN2
    from ganspace_b200.models.biggan import BigGAN
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    if name == "StyleGAN2":
        model = StyleGAN2(dev, cls, random_init=1234, use_w=space == "W")
    else:
        model = BigGAN(dev, int(name.split("-")[1]), cls, random_init=1234)
    model.eval()
    return InstrumentedModel(model)


def _timed(fns, reps):
    """Warm-up once, then ``reps`` alternated timed runs of each; returns (times, outputs of the warm-up)."""
    import torch
    outs = {key: fn() for key, fn in fns}
    times = {key: [] for key, _ in fns}
    for _ in range(reps):
        for key, fn in fns:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
    return times, outs


def _activation_workload(wl, reps, dev, gpu):
    import numpy as np
    import torch
    from ganspace_b200.strips import create_strip, create_strip_centered
    from act_strip_reference import reference_act_strip

    name, cls, layer, space, n_comp, n_frames, n_lat, centred = ACT_WORKLOADS[wl]
    inst = _act_inst(name, cls, space, dev)
    model = inst.model
    lats = [model.sample_latent(1, seed=100 + i).reshape(1, -1) for i in range(n_lat)]
    many = model.sample_latent(1000, seed=5)
    inst.retain_layer(layer)
    with torch.no_grad():
        model.partial_forward(many, layer)
    acts = inst.retained_layer(layer).clone().reshape(1000, -1)
    inst.close()
    W = acts.shape[1]
    mean = acts.mean(0, keepdim=True)
    g = torch.Generator().manual_seed(11)
    comps = (torch.randn(n_comp, W, generator=g) / np.sqrt(W)).to(dev)
    stdev = acts.std(0).mean() * torch.linspace(2.0, 0.5, n_comp, device=dev)
    sigma = 2.0

    def reference():
        return [reference_act_strip(inst, "activation", layer, lats, comps[c:c + 1], None, stdev[c], None, mean if centred else None,
                                    None, sigma, 0, -1, n_frames, centred) for c in range(n_comp)]

    def ours():
        if centred:
            return create_strip_centered(inst, "activation", layer, lats, comps, None, stdev, None, mean, None, sigma, 0, -1,
                                         n_frames, per_component=True)
        return create_strip(inst, "activation", layer, lats, comps, None, stdev, None, sigma, 0, -1, n_frames, per_component=True)

    times, outs = _timed((("reference", reference), ("strips", ours)), reps)
    diff = max(float(np.abs(a - b).max()) for ca, cb in zip(outs["reference"], outs["strips"]) for sa, sb in zip(ca, cb)
               for a, b in zip(sa, sb))
    n = n_comp * n_frames * n_lat
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"workload": wl, "model": f"{name}-{cls}", "layer": layer, "space": space, "mode": "activation",
                      "centred": centred, "frames": n, "res": int(outs["strips"][0][0][0].shape[0]),
                      "reference_frames_per_s": n / med["reference"], "strips_frames_per_s": n / med["strips"],
                      "speedup": med["reference"] / med["strips"], "reference_s": times["reference"], "strips_s": times["strips"],
                      "max_abs_frame_diff": diff, "gpu": gpu}), flush=True)
    inst.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(list(WORKLOADS) + list(ACT_WORKLOADS)))
    args = ap.parse_args()
    import numpy as np
    import torch
    from ganspace_b200.strips import create_strip_centered
    from strip_reference import reference_strip

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    gpu = _gpu_info()
    for wl in args.workloads.split(","):
        if wl in ACT_WORKLOADS:
            _activation_workload(wl, args.reps, dev, gpu)
            torch.cuda.empty_cache()
            continue
        name, cls, n_comp, n_frames, n_lat = WORKLOADS[wl]
        inst = _inst(name, cls, dev)
        model = inst.model
        lats = [model.sample_latent(1, seed=100 + i).reshape(1, -1) for i in range(n_lat)]
        many = model.sample_latent(1000, seed=5)
        mean = many.mean(0, keepdim=True)
        g = torch.Generator().manual_seed(11)
        comps = (torch.randn(n_comp, 512, generator=g) / np.sqrt(512)).to(dev)
        stdev = many.std(0).mean() * torch.linspace(2.0, 0.5, n_comp, device=dev)
        sigma = 2.0

        def reference():
            return [reference_strip(model, lats, comps[c:c + 1], stdev[c], mean, sigma, 0, -1, n_frames, True) for c in range(n_comp)]

        def ours():
            return create_strip_centered(inst, "latent", None, lats, None, comps, None, stdev, None, mean, sigma, 0, -1, n_frames,
                                         per_component=True)
        n = n_comp * n_frames * n_lat
        times = {"reference": [], "strips": []}
        outs = {}
        for fn in (reference, ours):                    # warm-up: every shape of the timed runs
            outs[fn.__name__] = fn()
        for _ in range(args.reps):
            for key, fn in (("reference", reference), ("strips", ours)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[key].append(time.perf_counter() - t0)
        diff = max(float(np.abs(a - b).max()) for ca, cb in zip(outs["reference"], outs["ours"]) for sa, sb in zip(ca, cb)
                   for a, b in zip(sa, sb))
        med = {k: float(np.median(v)) for k, v in times.items()}
        print(json.dumps({"workload": wl, "model": f"{name}-{cls}", "frames": n, "res": int(model.sample_np(lats[0]).shape[0]),
                          "reference_frames_per_s": n / med["reference"], "strips_frames_per_s": n / med["strips"],
                          "speedup": med["reference"] / med["strips"], "reference_s": times["reference"],
                          "strips_s": times["strips"], "max_abs_frame_diff": diff, "gpu": gpu}), flush=True)
        inst.close()
        del inst, model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
