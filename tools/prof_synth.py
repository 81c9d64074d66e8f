"""Timing of the config-5 pieces on one GPU: synthesis chain to convs.4 and the large-d IPCA step (CUDA events).
usage: python tools/prof_synth.py [n_samples_per_batch=2000] [steps=3]"""
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from ganspace_b200 import _native                     # noqa: E402
from ganspace_b200.models import StyleGAN2            # noqa: E402


def ev_time(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    nb = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    dev = torch.device("cuda:0")
    m = StyleGAN2(dev, "ffhq", random_init=1234)
    m.use_w()
    w = m.sample_latent(nb, seed=1)
    for layer, gf in (("conv1", 0.0755), ("convs.1", 0.453), ("convs.3", 1.963), ("convs.4", 3.171)):
        d = m._synthesis(m.synthesis_layer_names().index(layer) + 1).out_dims(m.synthesis_layer_names().index(layer) + 1)
        out = torch.empty((nb, d), dtype=torch.float32, device=dev)
        ms = ev_time(lambda: m.activations_into(w, layer, out))
        print(f"synthesis -> {layer}: n={nb} {ms:.2f} ms  {nb / ms * 1e3:.0f} samples/s  {nb * gf / ms:.1f} TFLOP/s (algorithmic)", flush=True)
    m.check_numerics()
    d, c = 512 * 32 * 32, 80
    big = _native.BigIPCA(d, c, nb, dev)
    rows = big.batch_rows(nb)
    for k in range(steps + 1):
        m.activations_into(m.sample_latent(nb, seed=100 + k), "convs.4", rows)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        big.step(nb)
        e1.record()
        torch.cuda.synchronize()
        print(f"bigd step {k} (direct): {e0.elapsed_time(e1):.2f} ms", flush=True)
    out = big.export()
    print("singular values head:", out["singular_values"][:5].cpu().numpy(), "ratio sum", float(out["explained_variance_ratio"].sum()))
    g = out["components"].double()
    print("orthonormality of components:", float((g @ g.T - torch.eye(c, dtype=torch.float64, device=dev)).abs().max()))
    print("peak memory GB:", torch.cuda.max_memory_allocated() / 1e9)


if __name__ == "__main__":
    t = time.time()
    main()
    print("wall", time.time() - t)
