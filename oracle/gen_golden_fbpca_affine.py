"""ORACLE -- generator of the --est fbpca fixtures on BigGAN-512 generator.gen_z (tests/golden/fbpca_{d,e}_*.npz).

Runs the UNMODIFIED reference (decomposition.get_or_compute -> estimators.FacebookPCAEstimator) on the CPU, by the
ref_harness recipe, with oracle/fbpca_affine_oracle.py (fbpca.pca with both of its randomized branches) installed as
``sys.modules['fbpca']``.
BigGAN-512 husky, random init 4321 (the weights of the ipca fixture c4s_biggan512_husky_genz_n4000_b1000_c16.npz),
layer 'generator.gen_z', B = 1000 (NB = 2000, so the stacked matrix ends in zero rows):
  (d) N = 32000, c = 16: [34000, 32768], fbpca's tall randomized branch; l = 32 is below the rank of the centred samples
      (129), so its range finder sees a strict subspace
  (e) N = 4000, c = 80: [6000, 32768], fbpca's wide randomized branch; l = 160 covers the rank, so its result is the exact
      top-80 PCA of the samples

The activation-space arrays (act_comp [c, 32768], act_mean) are stored as coefficients over gen_z's own 129 columns
(fbpca_affine_oracle.encode_span, with each row's residual); the tests rebuild them with decode_span.

Usage:  python oracle/gen_golden_fbpca_affine.py
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
    ("fbpca_d_biggan512_husky_genz_n32000_b1000_c16.npz", 32_000, 16),
    ("fbpca_e_biggan512_husky_genz_n4000_b1000_c80.npz", 4_000, 80),
]


def main():
    sys.path.insert(0, str(REPO))
    from oracle import fbpca_affine_oracle, ganspace_oracle, ref_harness
    sys.modules["fbpca"] = fbpca_affine_oracle
    ref = ref_harness.import_reference()
    assert ref.estimators.fbpca is fbpca_affine_oracle
    OUT.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cpu")
    only = sys.argv[1:]
    params = ganspace_oracle.biggan_genz_random_init(4321)
    for fname, n, c in CASES:
        if only and fname not in only:
            continue
        m = ref_harness.rand_init_biggan512(ref, dev, "husky", 4321)
        inst = ref.wrappers.get_instrumented_model("BigGAN-512", "husky", "generator.gen_z", dev, model=m)
        cfg = ref.Config(model="BigGAN-512", layer="generator.gen_z", output_class="husky", estimator="fbpca",
                         n=n, batch_size=1_000, components=c)
        with tempfile.TemporaryDirectory() as tmp:
            path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True,
                                                    submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
            with np.load(path) as data:
                out = {k: data[k].copy() for k in data.files}
        assert np.array_equal(params["weight_orig"], m.model.generator.gen_z.weight_orig.detach().numpy())   # same init
        enc = fbpca_affine_oracle.encode_span(out, params)
        assert enc["act_comp_resid"].max() < 1e-4 and enc["act_mean_resid"].max() < 1e-5, \
            (enc["act_comp_resid"].max(), enc["act_mean_resid"].max())
        np.savez_compressed(OUT / fname, dump_name=np.array(path.name), **enc)
        inst.close()
        print("wrote", fname, path.name, "residuals", enc["act_comp_resid"].max(), enc["act_mean_resid"].max(), flush=True)


if __name__ == "__main__":
    main()
