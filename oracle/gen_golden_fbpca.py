"""ORACLE -- generator of the --est fbpca golden fixtures (tests/golden/fbpca_*.npz).

Runs the UNMODIFIED reference (decomposition.get_or_compute -> estimators.FacebookPCAEstimator) on the CPU, by the
ref_harness recipe, with oracle/fbpca_oracle.py installed as ``sys.modules['fbpca']`` (the fbpca package is not part of the
reference and is absent here; the restatement follows its published algorithm).  StyleGAN2 random-init weights (seed 1234),
layer 'style':
  (a) W space, N = 10 000, B = 1000, c = 32: randomized branch, 2000 zero rows
  (b) Z space, N = 5000, B = 500, c = 16: ragged (K NB = 6000 < N + NB = 7000: 1000 zero rows), with the regression
  (c) W space, N = 4000, B = 1000, c = 210: exact branch (l = 420 >= 512 / 1.25)

Usage:  python oracle/gen_golden_fbpca.py
"""
import sys
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
OUT = REPO / "tests" / "golden"

CASES = [
    ("fbpca_a_stylegan2_ffhq_style_w_n10000_b1000_c32.npz", dict(n=10_000, batch_size=1_000, components=32), True),
    ("fbpca_b_stylegan2_ffhq_style_z_n5000_b500_c16.npz", dict(n=5_000, batch_size=500, components=16), False),
    ("fbpca_c_stylegan2_ffhq_style_w_n4000_b1000_c210.npz", dict(n=4_000, batch_size=1_000, components=210), True),
]


def main():
    sys.path.insert(0, str(REPO))
    from oracle import fbpca_oracle, ref_harness
    sys.modules["fbpca"] = fbpca_oracle
    ref = ref_harness.import_reference()
    assert ref.estimators.fbpca is fbpca_oracle
    OUT.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cpu")
    for fname, kw, use_w in CASES:
        m = ref_harness.rand_init_stylegan2(ref, dev, "ffhq")
        inst = ref.wrappers.get_instrumented_model("StyleGAN2", "ffhq", "style", dev, model=m, use_w=use_w)
        cfg = ref.Config(model="StyleGAN2", layer="style", output_class="ffhq", estimator="fbpca", use_w=use_w, **kw)
        with tempfile.TemporaryDirectory() as tmp:
            path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True,
                                                    submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
            with np.load(path) as data:
                out = {k: data[k].copy() for k in data.files}
        np.savez_compressed(OUT / fname, dump_name=np.array(path.name), **out)
        inst.close()
        print("wrote", fname, path.name)


if __name__ == "__main__":
    main()
