"""ORACLE -- BigGAN-deep conditional-BatchNorm row-layer fixtures (tests/golden/), produced by the UNMODIFIED reference on the CPU
(oracle/ref_harness.py).

The row layers are the bias-free spectral-norm linears ``generator.layers.k.bn_j.scale`` / ``.offset`` of every GenBlock (112 for
BigGAN-512, 80 for BigGAN-128).  Weights as in gen_golden_biggan_synth.py: ``ref_harness.rand_init_biggan512`` (random init under
torch.manual_seed(4321)) and, for 128, the same recipe with the reference's default ``BigGANConfig``; then
``synthesis_fill(net, 4321)``.

  R1  biggan_stylespace_known_answers.npz
        (a) the rows of every row layer of BigGAN-512, retained from the reference's ``forward`` for two seeded latents and for a
            list of 15 distinct latents (one per layer), and of BigGAN-128 for the two seeded latents: per layer a strided
            sub-sample of at most 64 channels (every C // 64-th) and, per sample, the fp64 sum and sum of squares of the whole row.
            One array per model and latent set: ``r{res}_{z|list}_sub`` [2, sum of the sub-sample widths] holds the layers'
            sub-samples side by side in the order of ``r{res}_names`` (widths ``r{res}_widths``), ``..._sum`` / ``..._sq`` are
            [layers, 2] (``biggan_stylespace_oracle.known_rows`` unpacks them);
        (b) BigGAN-512 ``forward`` images of the two seeded latents with
              - ``edit_layer(EDIT_SCALE, offset=[1, C])``,
              - ``edit_layer(EDIT_OFFSET, offset=[2, C])`` (one offset per sample),
            the edits at the scale of the layer's rows,
              - ``edit_layer(EDIT_ABLATE, ablation=0.5, replacement=[C])``,
            each sub-sampled to 32^2 (every 16th pixel) plus per-sample sums, with the output of the block before the edited one
            retained in the same call (its per-sample sums of squares)
  R2  bs_biggan512_husky_l0bn1scale_z_n4000_b1000_c16.npz    get_or_compute on generator.layers.0.bn_1.scale (C = 512), ipca
  R3  bs_biggan512_husky_l1bn0offset_z_n4000_b1000_c16_fbpca.npz
                                                             get_or_compute on generator.layers.1.bn_0.offset (C = 2048), fbpca, with
                                                             oracle/fbpca_oracle.py installed as ``sys.modules['fbpca']``

Usage:  python oracle/gen_golden_biggan_stylespace.py [r1] [r2] [r3]   (a few minutes of CPU time; about 0.4 MB in all)
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
from oracle.biggan_stylespace_oracle import row_stride          # noqa: E402

OUT = REPO / "tests" / "golden"
SEED = 4321
N = 2
EDIT_SCALE = "generator.layers.11.bn_2.scale"         # C = 64
EDIT_OFFSET = "generator.layers.13.bn_1.offset"       # C = 32
EDIT_ABLATE = "generator.layers.10.bn_0.offset"       # C = 512, after the SelfAttn at generator.layers.8


def _store_rows(ka, k, feats, names):
    """The rows of ``names`` (retained features), packed as the module docstring describes."""
    ka[f"{k}_sub"] = np.concatenate([feats[n][:, ::row_stride(feats[n].shape[1])].numpy() for n in names], axis=1)
    ka[f"{k}_sum"] = np.stack([feats[n].double().sum(dim=1).numpy() for n in names])
    ka[f"{k}_sq"] = np.stack([feats[n].double().pow(2).sum(dim=1).numpy() for n in names])


def row_layer_names(model):
    from models import biggan
    return [f"generator.layers.{k}.bn_{j}.{kind}" for k, layer in enumerate(model.generator.layers)
            if isinstance(layer, biggan.GenBlock) for j in range(4) for kind in ("scale", "offset")]


def _models(ref, dev):
    from ganspace_b200.models.biggan import synthesis_fill
    from models import biggan
    m = rh.rand_init_biggan512(ref, dev, "husky", SEED)
    synthesis_fill(m.model, SEED)
    m.eval()

    class RandInit128(ref.wrappers.BigGAN):
        def load_model(self, name):
            torch.manual_seed(SEED)
            self.model = biggan.BigGAN(biggan.BigGANConfig()).to(self.device)

    m128 = RandInit128(dev, 128, "husky")
    synthesis_fill(m128.model, SEED)
    m128.eval()
    return m, m128


def known_answers():
    ref = rh.import_reference()
    from models import biggan
    from netdissect.nethook import InstrumentedModel
    dev = torch.device("cpu")
    torch.set_grad_enabled(False)
    ka = {}
    m, m128 = _models(ref, dev)
    z = torch.from_numpy(biggan.truncated_noise_sample(truncation=1.0, batch_size=N, seed=21))
    z_list = [torch.from_numpy(biggan.truncated_noise_sample(truncation=1.0, batch_size=N, seed=200 + i))
              for i in range(m.model.n_latents)]
    ka["z"], ka["z_list"] = z.numpy(), np.stack([t.numpy() for t in z_list])

    for tag, model, res in (("512", m, 512), ("128", m128, 128)):
        names = row_layer_names(model.model)
        inst = InstrumentedModel(model)          # (get_instrumented_model's shape pass would run one partial_forward per layer)
        inst.retain_layers(names)
        ka[f"r{tag}_names"] = np.array(names)
        ka[f"r{tag}_widths"] = np.array([getattr(model.model.get_submodule(n.rsplit(".", 1)[0]), "num_features") for n in names])
        model.forward(z)
        _store_rows(ka, f"r{tag}_z", inst.retained_features(), names)
        if tag == "512":
            full = {n: inst.retained_layer(n).double().numpy().copy() for n in names}
            model.forward(z_list)
            _store_rows(ka, f"r{tag}_list", inst.retained_features(), names)
        inst.close()

    def img(tag, x):
        ka[f"img_{tag}_sub"] = x[:, :, ::16, ::16].contiguous().numpy()
        ka[f"img_{tag}_sum"] = x.double().sum(dim=(1, 2, 3)).numpy()

    # edits at the scale of the layer's own rows (``full``: BigGAN-512's rows at z) (random-init rows reach a few hundred), so that each one shows in the image
    rng = np.random.RandomState(77)
    rms = lambda name: float(np.sqrt((full[name] ** 2).mean()))
    width = lambda name: full[name].shape[1]
    edits = {
        "scale": (EDIT_SCALE, dict(offset=(rms(EDIT_SCALE) * rng.standard_normal((1, width(EDIT_SCALE)))).astype(np.float32))),
        "offset": (EDIT_OFFSET, dict(offset=(2 * rms(EDIT_OFFSET) * rng.standard_normal((N, width(EDIT_OFFSET)))).astype(np.float32))),
        "ablate": (EDIT_ABLATE, dict(ablation=0.5, replacement=(
            2 * rms(EDIT_ABLATE) * rng.standard_normal(width(EDIT_ABLATE))).astype(np.float32))),
    }
    for tag, (layer, kw) in edits.items():
        prev = f"generator.layers.{int(layer.split('.')[2]) - 1}"
        inst = InstrumentedModel(m)
        inst.retain_layers([layer, prev])
        inst.edit_layer(layer, **{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()})
        img(tag, m.forward(z))
        ka[f"prev_{tag}_sq"] = inst.retained_layer(prev).double().pow(2).sum(dim=(1, 2, 3)).numpy()
        for k, v in kw.items():
            ka[f"edit_{tag}_{k}"] = np.asarray(v)
        inst.close()
    np.savez_compressed(OUT / "biggan_stylespace_known_answers.npz", **ka)
    print("wrote biggan_stylespace_known_answers.npz", (OUT / "biggan_stylespace_known_answers.npz").stat().st_size, "bytes")


def end_to_end(layer, estimator, out_name, n=4_000, b=1_000, c=16):
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m, _ = _models(ref, dev)
    inst = ref.wrappers.get_instrumented_model("BigGAN-512", "husky", layer, dev, model=m)
    cfg = ref.Config(model="BigGAN-512", layer=layer, output_class="husky", estimator=estimator, n=n, batch_size=b, components=c)
    t0 = time.time()
    with tempfile.TemporaryDirectory() as tmp:
        path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True,
                                                submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
        with np.load(path) as data:
            out = {k: data[k].copy() for k in data.files}
        name = path.name
    print(f"{layer} {estimator}: {time.time() - t0:.0f} s", flush=True)
    inst.close()
    np.savez_compressed(OUT / out_name, dump_name=np.array(name), **out)


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"r1", "r2", "r3"}
    if "r3" in which:
        from oracle import fbpca_oracle
        sys.modules["fbpca"] = fbpca_oracle                 # before the reference's estimators module imports it
    if "r1" in which:
        known_answers()
    if "r2" in which:
        end_to_end("generator.layers.0.bn_1.scale", "ipca", "bs_biggan512_husky_l0bn1scale_z_n4000_b1000_c16.npz")
    if "r3" in which:
        end_to_end("generator.layers.1.bn_0.offset", "fbpca", "bs_biggan512_husky_l1bn0offset_z_n4000_b1000_c16_fbpca.npz")
