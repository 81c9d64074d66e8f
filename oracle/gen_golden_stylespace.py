"""ORACLE -- StyleGAN2 style-space fixtures (tests/golden/), produced by the UNMODIFIED reference on CPU (oracle/ref_harness.py).

The S layers are the 26 modulation layers (``EqualLinear``) of an ffhq-1024 generator: ``conv1.conv.modulation``,
``convs.k.conv.modulation``, ``to_rgb1.conv.modulation`` and ``to_rgbs.j.conv.modulation``.  Random init 1234, with the
non-zero NoiseInjection weights, activation biases and ToRGB biases of gen_golden_r2.py's G11.

  S1  stylespace_known_answers.npz   (a) the modulation output of every S layer, retained from the reference's
                                     ``forward``, for four seeded Z latents and for one list of 18 per-layer Z latents (2 samples);
                                     (b) ``forward`` images with ``edit_layer('convs.5.conv.modulation', offset=[2, 512])`` and with
                                     ``edit_layer('to_rgbs.2.conv.modulation', ablation=0.5, replacement=[512])`` (stored ::16 plus sums)
  S2  c6_stylegan2_ffhq_convs1mod_z_n4000_b500_c16.npz    get_or_compute on convs.1.conv.modulation, Z space with regression
  S3  c6_stylegan2_ffhq_torgb1mod_w_n4000_b500_c16.npz    get_or_compute on to_rgb1.conv.modulation, W space

Usage:  python oracle/gen_golden_stylespace.py [s1] [s2] [s3]
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
from oracle.gen_golden import perturb_synthesis  # noqa: E402

OUT = REPO / "tests" / "golden"
CONV_NAMES = ["conv1"] + [f"convs.{i}" for i in range(16)]
RGB_NAMES = ["to_rgb1"] + [f"to_rgbs.{i}" for i in range(8)]
S_NAMES = [f"{n}.conv.modulation" for n in CONV_NAMES + RGB_NAMES]


def perturbed_model(ref, dev):
    """G11's model: random init 1234, perturbed noise weights / activation biases on every StyledConv, non-zero ToRGB biases."""
    m = rh.rand_init_stylegan2(ref, dev, "ffhq", 1234)
    perturb_synthesis(m.model, CONV_NAMES)
    mods = dict(m.model.named_modules())
    with torch.no_grad():
        for i, nme in enumerate(RGB_NAMES):
            mods[nme].bias.copy_(0.05 * torch.tensor([1.0, -2.0, 3.0]).view(1, 3, 1, 1) * (i + 1))
    return m


def _img(ka, key, img):
    ka[f"{key}_sub"] = img[:, :, ::16, ::16].copy()          # every 16th pixel each way (64 x 64) keeps the fixture small
    ka[f"{key}_sum"] = np.array([img.astype(np.float64).sum(), (img.astype(np.float64) ** 2).sum()])


def known_answers():
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = perturbed_model(ref, dev)
    inst = ref.wrappers.get_instrumented_model("StyleGAN2", "ffhq", S_NAMES[0], dev, model=m, use_w=False)
    inst.retain_layers(S_NAMES[1:])
    m.use_z()
    ka = dict(s_names=np.array(S_NAMES))
    z4 = m.sample_latent(4, seed=31)
    with torch.no_grad():
        img = m.forward(z4).numpy()
    ka["z4"] = z4.numpy()
    feats = inst.retained_features()
    for name in S_NAMES:
        ka["s4_" + name.replace(".", "_")] = feats[name].numpy().copy()
    _img(ka, "img4", img)
    z18 = [m.sample_latent(2, seed=40 + k) for k in range(18)]
    with torch.no_grad():
        m.forward(z18)
    ka["z18"] = torch.stack(z18).numpy()                                       # [18, 2, 512]
    feats = inst.retained_features()
    for name in S_NAMES:
        ka["s18_" + name.replace(".", "_")] = feats[name].numpy().copy()

    # (b) edits; the images use the first two latents of z4
    z2 = z4[:2]
    rng = np.random.RandomState(77)
    offset = (0.5 * rng.standard_normal((2, 512))).astype(np.float32)
    inst.edit_layer("convs.5.conv.modulation", offset=torch.from_numpy(offset))
    with torch.no_grad():
        _img(ka, "img_offset", m.forward(z2).numpy())
    inst.remove_edits()
    replacement = (1.0 + 0.3 * rng.standard_normal(512)).astype(np.float32)
    inst.edit_layer("to_rgbs.2.conv.modulation", ablation=0.5, replacement=torch.from_numpy(replacement))
    with torch.no_grad():
        _img(ka, "img_ablate", m.forward(z2).numpy())
    inst.remove_edits()
    ka["edit_offset"], ka["edit_replacement"] = offset, replacement
    inst.close()
    np.savez_compressed(OUT / "stylespace_known_answers.npz", **ka)
    print("wrote stylespace_known_answers.npz")


def end_to_end(layer, use_w, out_name, n=4_000, b=500, c=16):
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = perturbed_model(ref, dev)
    inst = ref.wrappers.get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=m, use_w=use_w)
    cfg = ref.Config(model="StyleGAN2", layer=layer, output_class="ffhq", estimator="ipca", use_w=use_w, n=n, batch_size=b,
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
    which = set(sys.argv[1:]) or {"s1", "s2", "s3"}
    if "s1" in which:
        known_answers()
    if "s2" in which:
        end_to_end("convs.1.conv.modulation", False, "c6_stylegan2_ffhq_convs1mod_z_n4000_b500_c16.npz")
    if "s3" in which:
        end_to_end("to_rgb1.conv.modulation", True, "c6_stylegan2_ffhq_torgb1mod_w_n4000_b500_c16.npz")
