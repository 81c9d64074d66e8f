"""StyleGAN (v1, random init 1234 + synthesis_fill 7) on one GPU:

  * ``forward`` images/s at batch 1 / 8 / 32 for ffhq (1024) and bedrooms (256), alternating with the plain-PyTorch fp32 forward of
    the same equations (oracle/stylegan_oracle.py::layer_torch: cuDNN convs, TF32 off) on the same GPU;
  * the synthesis chain's achieved rate against the useful work counted as the reference convolves (at output resolution), and the
    CUDA-event time of each block (cumulative runs to block k, differenced);
  * get_or_compute time for g_mapping in W space (N = 10^6, B = 10^4, c = 80) and for g_synthesis.blocks.32x32 (N = 20,000,
    B = 500, c = 80).
Prints one JSON line (with the card's name, power limit and max SM clock) and writes it to --out.

    python tools/bench_stylegan.py [--reps 3] [--out FILE] [--skip-decomp]
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


def useful_flops(model):
    """Multiply-adds x 2 of the convolutions as the reference runs them (3x3 at the output resolution, torgb) plus the blur."""
    total = 0
    for conv, epi, up, r in model.model.g_synthesis.layer_modules():
        if conv is not None:
            co, ci = conv.weight.shape[:2]
            total += 2 * r * r * co * ci * 9 + (2 * r * r * co * 9 if up else 0)
    r, c = model.resolution, model.model.g_synthesis.torgb.weight.shape[1]
    return total + 2 * r * r * 3 * c


def hbm_bytes(packed, n):
    """Bytes the chain moves through HBM at least: per layer the tap plane Y written and read, A written and read, the operand
    written (fp16 hi/lo) and read by the next GEMM, the up-conv output U written and read (fp32)."""
    total = 0
    for (r, c), d in zip(packed.shapes, packed.desc):
        hw, hw_in = r * r, (r // 2 if d.upsample else r) ** 2
        if d.conv_weight:
            total += 2 * 4 * hw_in * ((9 * c + 31) // 32 * 32)
        total += 2 * 4 * hw * c + 2 * 4 * hw * c + (2 * 4 * hw * c if d.upsample else 0)
    return total * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-decomp", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch
    from ganspace_b200.models import StyleGAN, get_instrumented_model, stylegan
    from oracle import stylegan_oracle as so
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    res = {"gpu": _gpu_info()}
    for cls in ("bedrooms", "ffhq"):
        m = StyleGAN(dev, cls, random_init=1234)
        stylegan.synthesis_fill(m.model, 7)
        m.use_w()
        sd = {k: v.detach().float() for k, v in m.model.state_dict().items()}
        noise = {r: torch.from_numpy(v).to(dev) for r, v in so.fixed_noise(m.resolution).items()}
        lays = so.layers(sd, m.resolution)

        def baseline(w):
            x = None
            for _, conv, epi, up, r in lays:
                x = so.layer_torch(x, w, sd, conv, epi, up, noise[r])
            W = sd["g_synthesis.torgb.weight"]
            return 0.5 * (torch.nn.functional.conv2d(x, W / float(np.sqrt(W.shape[1])), sd["g_synthesis.torgb.bias"]) + 1)

        flops, packed = useful_flops(m), m.model.g_synthesis.packed()
        out = {"useful_gflop_per_image": flops / 1e9}
        for bs in (1, 8, 32):
            w = m.sample_latent(bs, seed=bs)
            with torch.no_grad():
                err = float((m.forward(w) - baseline(w)).abs().max())
                ours = base = 0.0
                for _ in range(args.reps):                 # alternating
                    ours += _event_ms(lambda: m.forward(w), 3)
                    base += _event_ms(lambda: baseline(w), 3)
            ours, base = ours / args.reps, base / args.reps
            chain = _event_ms(lambda: packed.forward(w, packed.n_layers, want_act=False, want_rgb=True), 3)
            out[f"b{bs}"] = dict(images_per_s=1e3 * bs / ours, ms=ours, baseline_images_per_s=1e3 * bs / base, baseline_ms=base,
                                 max_abs_diff_vs_baseline=err, chain_ms=chain, chain_tflops=flops * bs / chain / 1e9,
                                 flop_bound_share=flops * bs / (989e12 / 3) / (chain / 1e3),
                                 hbm_bound_share=hbm_bytes(packed, bs) / 3.35e12 / (chain / 1e3))
        w = m.sample_latent(8, seed=1)
        prev, per_block = 0.0, {}
        for k, name in enumerate(m.model.block_names()):
            t = _event_ms(lambda: packed.forward(w, 2 * (k + 1)), 3)
            per_block[name.rsplit(".", 1)[1]] = t - prev
            prev = t
        out["block_ms_b8"] = per_block
        res[cls] = out
        print(cls, json.dumps(out), flush=True)
        if cls == "bedrooms":
            del m, packed
            torch.cuda.empty_cache()
    if not args.skip_decomp:
        from ganspace_b200.config import Config
        from ganspace_b200.decomposition import get_or_compute
        for layer, use_w, n, b in (("g_mapping", True, 1_000_000, 10_000), ("g_synthesis.blocks.32x32", False, 20_000, 500)):
            inst = get_instrumented_model("StyleGAN", "ffhq", layer, dev, model=m, use_w=use_w)
            cfg = Config(model="StyleGAN", layer=layer, output_class="ffhq", components=80, n=n, batch_size=b, estimator="ipca",
                         use_w=use_w)
            times = []
            for _ in range(2):
                with tempfile.TemporaryDirectory() as tmp:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t0)
            res[f"get_or_compute_{layer}_{'w' if use_w else 'z'}_n{n}_b{b}_c80_s"] = times
            inst.close()
            m.use_z()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
