"""ORACLE -- StyleGAN (v1) style-space fixtures (tests/golden/), produced by the UNMODIFIED reference on CPU (oracle/ref_harness.py).

The style layers are the StyleMod linears ``g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin`` (18 for ffhq-1024, 14 for
bedrooms-256).  Weights as in gen_golden_stylegan.py: ``torch.manual_seed(1234); StyleGAN_G(res)``, then
``synthesis_fill(net, 7)``.

  V1  stylegan_stylespace_known_answers.npz
        (a) the rows of every style layer of ffhq and of bedrooms, retained from the reference's ``forward``, for four seeded Z
            latents and for the 18 distinct W latents of ``stylegan_oracle.w18_latents`` (4 samples);
        (b) ffhq ``forward`` images of the first two Z latents with ``edit_layer('g_synthesis.blocks.16x16.epi2.style_mod.lin',
            offset=[2, 1024])`` and with ``edit_layer('g_synthesis.blocks.4x4.epi1.style_mod.lin', ablation=0.5,
            replacement=[1024])``, stored as every 16th pixel each way plus full-image sums
  V2  sv_stylegan_ffhq_8x8epi1lin_z_n4000_b500_c16.npz     get_or_compute on blocks.8x8.epi1.style_mod.lin, Z space (regression)
  V3  sv_stylegan_ffhq_32x32epi2lin_w_n4000_b500_c16.npz   get_or_compute on blocks.32x32.epi2.style_mod.lin, W space

Usage:  python oracle/gen_golden_stylegan_stylespace.py [v1] [v2] [v3]
"""
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
from oracle import ref_harness as rh          # noqa: E402
from oracle.gen_golden_stylegan import rand_init_stylegan          # noqa: E402
from oracle.stylegan_oracle import w18_latents          # noqa: E402
from oracle.stylegan_stylespace_oracle import style_layer_names          # noqa: E402

OUT = REPO / "tests" / "golden"
OFFSET_LAYER = "g_synthesis.blocks.16x16.epi2.style_mod.lin"
ABLATE_LAYER = "g_synthesis.blocks.4x4.epi1.style_mod.lin"


def key(name):
    return name[len("g_synthesis.blocks."):].replace(".", "_")


def _img(ka, k, img):
    ka[f"{k}_sub"] = img[:, :, ::16, ::16].copy()
    ka[f"{k}_sum"] = np.array([img.astype(np.float64).sum(), (img.astype(np.float64) ** 2).sum()])


def known_answers():
    ref = rh.import_reference()
    dev = torch.device("cpu")
    ka = {}
    for cls, res in (("ffhq", 1024), ("bedrooms", 256)):
        t0 = time.time()
        m = rand_init_stylegan(ref, dev, cls)
        names = style_layer_names(res)
        inst = ref.wrappers.get_instrumented_model("StyleGAN", cls, names, dev, model=m)
        m.use_z()
        z4 = m.sample_latent(4, seed=31)
        ka[f"{cls}_z4"] = z4.numpy()
        with torch.no_grad():
            img4 = m.forward(z4).numpy()
        for name, rows in inst.retained_features().items():
            ka[f"{cls}_z4_{key(name)}"] = rows.numpy().copy()
        m.use_w()
        with torch.no_grad():
            m.forward([torch.from_numpy(w) for w in w18_latents()])
        m.use_z()
        for name, rows in inst.retained_features().items():
            ka[f"{cls}_w18_{key(name)}"] = rows.numpy().copy()
        if cls == "ffhq":
            _img(ka, "img4", img4[:2])
            z2 = z4[:2]
            rng = np.random.RandomState(77)
            offset = (0.5 * rng.standard_normal((2, 1024))).astype(np.float32)
            inst.edit_layer(OFFSET_LAYER, offset=torch.from_numpy(offset))
            with torch.no_grad():
                _img(ka, "img_offset", m.forward(z2).numpy())
            inst.remove_edits()
            replacement = (0.3 * rng.standard_normal(1024)).astype(np.float32)
            inst.edit_layer(ABLATE_LAYER, ablation=0.5, replacement=torch.from_numpy(replacement))
            with torch.no_grad():
                _img(ka, "img_ablate", m.forward(z2).numpy())
            inst.remove_edits()
            ka["edit_offset"], ka["edit_replacement"] = offset, replacement
        inst.close()
        print(cls, f"{time.time() - t0:.0f} s", flush=True)
    np.savez_compressed(OUT / "stylegan_stylespace_known_answers.npz", **ka)
    print("wrote stylegan_stylespace_known_answers.npz")


def end_to_end(layer, use_w, out_name, n=4_000, b=500, c=16):
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = rand_init_stylegan(ref, dev, "ffhq")
    inst = ref.wrappers.get_instrumented_model("StyleGAN", "ffhq", layer, dev, model=m, use_w=use_w)
    cfg = ref.Config(model="StyleGAN", layer=layer, output_class="ffhq", estimator="ipca", use_w=use_w, n=n, batch_size=b,
                     components=c)
    t0 = time.time()
    with tempfile.TemporaryDirectory() as tmp:
        path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
        with np.load(path) as data:
            out = {k: data[k].copy() for k in data.files}
        name = path.name
    print(f"{layer}: {time.time() - t0:.0f} s", flush=True)
    inst.close()
    np.savez_compressed(OUT / out_name, dump_name=np.array(name), **out)


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"v1", "v2", "v3"}
    if "v1" in which:
        known_answers()
    if "v2" in which:
        end_to_end("g_synthesis.blocks.8x8.epi1.style_mod.lin", False, "sv_stylegan_ffhq_8x8epi1lin_z_n4000_b500_c16.npz")
    if "v3" in which:
        end_to_end("g_synthesis.blocks.32x32.epi2.style_mod.lin", True, "sv_stylegan_ffhq_32x32epi2lin_w_n4000_b500_c16.npz")
