"""ORACLE -- StyleGAN (v1) golden fixtures (tests/golden/), produced by the UNMODIFIED reference on the host CPU.

  stylegan_known_answers.npz      for ffhq (1024) and bedrooms (256), 4 seeded latents: z, W, every block's output (strided
                                  sub-sample of at most 8 channels x 16 x 16 + per-sample sums and sums of squares) and the image
                                  (32 x 32 sub-sample + per-sample sums) of StyleGAN.forward in Z mode, the same for one forward on a
                                  list of 18 distinct W, init spot values and the state-dict keys
  sg_stylegan_ffhq_g_mapping_{z,w}_n4000_b500_c16.npz, sg_stylegan_ffhq_8x8_z_n4000_b500_c8.npz
                                  decomposition.get_or_compute at g_mapping (Z with the regression pass, W) and at
                                  g_synthesis.blocks.8x8 (d = 32,768; act_comp stored as float16)

The reference's StyleGAN wrapper is used as is except ``load_model`` (no network for the checkpoint): ``torch.manual_seed(1234);
StyleGAN_G(res)`` followed by ``ganspace_b200.models.stylegan.synthesis_fill(net, 7)``, which gives the biases, the constant and the
noise weights (zero or one in the reference's init) seeded values.

Usage:  python oracle/gen_golden_stylegan.py [ka] [e2e]
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
from oracle.stylegan_oracle import w18_latents          # noqa: E402
from ganspace_b200.models.stylegan import synthesis_fill          # noqa: E402

OUT = REPO / "tests" / "golden"
SEED, FILL = 1234, 7


def rand_init_stylegan(ref, device, outclass):
    stylegan = ref.wrappers.stylegan

    class RandInitStyleGAN(ref.wrappers.StyleGAN):
        def load_model(self):                      # replaces the checkpoint download / TF conversion (wrappers.py:311-347)
            torch.manual_seed(SEED)
            self.model = synthesis_fill(stylegan.StyleGAN_G(self.resolution), FILL).to(self.device)

    return RandInitStyleGAN(device, outclass)


def sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step].copy()


def sums(a):
    a = a.astype(np.float64).reshape(len(a), -1)
    return np.stack([a.sum(1), (a * a).sum(1)], 1)


def known_answers():
    ref = rh.import_reference()
    dev = torch.device("cpu")
    ka = {}
    for cls in ("ffhq", "bedrooms"):
        t0 = time.time()
        m = rand_init_stylegan(ref, dev, cls)
        names = [f"g_synthesis.blocks.{n}" for n in m.model._modules["g_synthesis"].blocks]
        sd = m.model.state_dict()
        ka[f"{cls}_state_dict_keys"] = np.array(list(sd))
        ka[f"{cls}_n_modules"] = np.array(len(list(m.model.named_modules())))
        for k in ("g_mapping.dense0.weight", "g_mapping.dense7.bias", "g_synthesis.torgb.weight", "g_synthesis.blocks.4x4.const",
                  f"{names[-1]}.conv1.weight", f"{names[-1]}.epi2.style_mod.lin.weight", f"{names[1]}.epi1.top_epi.noise.weight"):
            ka[f"{cls}_init_{k}"] = sd[k].reshape(-1)[:64].numpy().copy()
        z = m.sample_latent(4, seed=21)
        with torch.no_grad():
            ka[f"{cls}_z"] = z.numpy()
            ka[f"{cls}_w"] = m.model._modules["g_mapping"].forward(z).numpy()
        w18 = w18_latents()
        inst = ref.wrappers.get_instrumented_model("StyleGAN", cls, names, dev, model=m)
        for tag, run in (("z", lambda: m.forward(z)),
                         ("w18", lambda: (m.use_w(), m.forward([torch.from_numpy(w) for w in w18]))[1])):
            with torch.no_grad():
                img = run().numpy()
            m.use_z()
            for name, act in inst.retained_features().items():
                act = act.numpy()
                b = name.rsplit(".", 1)[1]
                ka[f"{cls}_{tag}_{b}_sub"] = sub(act)
                ka[f"{cls}_{tag}_{b}_sums"] = sums(act)
                ka[f"{cls}_{b}_shape"] = np.array(act.shape)
            step = max(1, img.shape[-1] // 32)
            ka[f"{cls}_{tag}_image_sub"] = img[:, :, ::step, ::step].copy()
            ka[f"{cls}_{tag}_image_sums"] = sums(img)
        inst.close()
        print(cls, f"{time.time() - t0:.0f} s", flush=True)
    np.savez_compressed(OUT / "stylegan_known_answers.npz", **ka)
    print("wrote stylegan_known_answers.npz", sum(v.nbytes for v in ka.values()) / 1e6, "MB raw")


def end_to_end(layer, use_w, c, n=4_000, b=500):
    ref = rh.import_reference()
    dev = torch.device("cpu")
    m = rand_init_stylegan(ref, dev, "ffhq")
    inst = ref.wrappers.get_instrumented_model("StyleGAN", "ffhq", layer, dev, model=m)
    cfg = ref.Config(model="StyleGAN", layer=layer, output_class="ffhq", estimator="ipca", use_w=use_w, n=n, batch_size=b, components=c)
    t0 = time.time()
    with tempfile.TemporaryDirectory() as tmp:
        path = ref.decomposition.get_or_compute(cfg, inst, force_recompute=True, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp))
        with np.load(path) as data:
            out = {k: data[k].copy() for k in data.files}
        name = path.name
    print(f"{layer} use_w={use_w}: {time.time() - t0:.0f} s", flush=True)
    inst.close()
    short = layer.rsplit(".", 1)[-1]
    if out["act_comp"].size > 100_000:
        out["act_comp_f16"] = out.pop("act_comp").astype(np.float16)
    np.savez_compressed(OUT / f"sg_stylegan_ffhq_{short}_{'w' if use_w else 'z'}_n{n}_b{b}_c{c}.npz", dump_name=np.array(name), **out)


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"ka", "e2e"}
    if "ka" in which:
        known_answers()
    if "e2e" in which:
        end_to_end("g_mapping", False, 16)
        end_to_end("g_mapping", True, 16)
        end_to_end("g_synthesis.blocks.8x8", False, 8)
