"""ORACLE -- ProGAN golden fixtures (tests/golden/), produced by the UNMODIFIED reference on the host CPU.

  progan_known_answers.npz                       every block's activation (strided sub-sample of at most 8 channels x 16 x 16
                                                 + sum / sum of squares of the whole tensor) and the image of ProGAN.forward
                                                 (stored ::8) for 4 seeded latents, random init (seed 1234)
  pg_progan_bedroom_layer4_n4000_b500_c8.npz     decomposition.get_or_compute at layer4 (d = 32,768) with the regression pass;
                                                 act_comp stored as float16 (0.5 MB instead of 1)

The reference's ProGAN wrapper is used as is except ``load_model`` (no network for the checkpoint): random weights as
oracle/progan_oracle.py::progan_random_init describes.

Usage:  python oracle/gen_golden_progan.py [ka] [e2e]
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

OUT = REPO / "tests" / "golden"
SEED = 1234


def rand_init_progan(ref, device, outclass="bedroom", seed=SEED):
    """The reference's ProGAN wrapper with random weights (load_model is the only override)."""
    proggan = ref.wrappers.proggan

    class RandInitProGAN(ref.wrappers.ProGAN):
        def load_model(self):                      # replaces the checkpoint download (wrappers.py:483-492)
            torch.manual_seed(seed)
            model = proggan.ProgressiveGenerator(resolution=256)
            with torch.no_grad():
                for m in model._modules.values():
                    m.conv.weight.copy_(torch.randn(m.conv.weight.shape))
            self.model = model.to(self.device)

    return RandInitProGAN(device, outclass)


def sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step].copy()


def known_answers():
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = rand_init_progan(ref, dev)
    names = list(m.model._modules)
    z = m.sample_latent(4, seed=21)
    ka = dict(z=z.numpy(), names=np.array(names))
    sd = m.model.state_dict()
    ka["state_dict_keys"] = np.array(list(sd))
    # spot values of the random init: the first conv weights and biases of three blocks (the init order is part of the contract)
    for name in ("layer1", "layer7", names[-1]):
        ka[f"init_{name}_w"] = sd[f"{name}.conv.weight"].reshape(-1)[:64].numpy().copy()
        ka[f"init_{name}_b"] = sd[f"{name}.wscale.b"].reshape(-1)[:3].numpy().copy()
    inst = ref.wrappers.get_instrumented_model("ProGAN", "bedroom", names, dev, model=m)
    with torch.no_grad():
        img = m.forward(z).numpy()
    for name, act in inst.retained_features().items():
        act = act.numpy()
        ka[f"act_{name}_sub"] = sub(act)
        ka[f"sum_{name}"] = np.array([act.astype(np.float64).sum(), (act.astype(np.float64) ** 2).sum()])
        ka[f"shape_{name}"] = np.array(act.shape)
    inst.close()
    ka["img_sub"] = img[:, :, ::8, ::8].copy()
    ka["img_sum"] = np.array([img.astype(np.float64).sum(), (img.astype(np.float64) ** 2).sum()])
    # partial_forward == forward at a hooked layer, in the reference itself
    inst = ref.wrappers.get_instrumented_model("ProGAN", "bedroom", "layer5", dev, model=m)
    with torch.no_grad():
        m.partial_forward(z, "layer5")
    assert np.array_equal(sub(inst.retained_features()["layer5"].numpy()), ka["act_layer5_sub"])
    inst.close()
    np.savez_compressed(OUT / "progan_known_answers.npz", **ka)
    print("wrote progan_known_answers.npz", {k: v.shape for k, v in ka.items() if k.endswith("_sub")})


def end_to_end(layer="layer4", n=4_000, b=500, c=8):
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = rand_init_progan(ref, dev)
    inst = ref.wrappers.get_instrumented_model("ProGAN", "bedroom", layer, dev, model=m)
    cfg = ref.Config(model="ProGAN", layer=layer, output_class="bedroom", estimator="ipca", use_w=False, n=n, batch_size=b, components=c)
    t0 = time.time()
    with tempfile.TemporaryDirectory() as tmp:
        path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
        with np.load(path) as data:
            out = {k: data[k].copy() for k in data.files}
        name = path.name
    print(f"{layer}: {time.time() - t0:.0f} s", flush=True)
    inst.close()
    out["act_comp_f16"] = out.pop("act_comp").astype(np.float16)
    np.savez_compressed(OUT / f"pg_progan_bedroom_{layer}_n{n}_b{b}_c{c}.npz", dump_name=np.array(name), **out)


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"ka", "e2e"}
    if "ka" in which:
        known_answers()
    if "e2e" in which:
        end_to_end()
