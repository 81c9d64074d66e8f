"""Known answers of BigGAN-deep synthesis from the UNMODIFIED reference on the CPU -> tests/golden/biggan_synthesis_known_answers.npz.

The reference wrapper (models/wrappers.py BigGAN) is built with ``ref_harness.rand_init_biggan512`` (random init under
torch.manual_seed(4321); only ``load_model`` is replaced) and, for 128, the same recipe with the reference's default
``BigGANConfig``.  A random init leaves the BatchNorm statistics tables, ``SelfAttn.gamma`` and ``generator.bn.weight`` / ``bias``
degenerate or undefined; ``ganspace_b200.models.biggan.synthesis_fill`` (seed 4321) gives both the reference model and ours the same
values for them.  Then, in eval mode (as get_instrumented_model leaves it):

  * init checksums of every state-dict tensor (fp64 sum and sum of squares);
  * ``partial_forward(z, 'generator.layers.14')`` with a forward hook on every ``generator.layers.k``: a strided sub-sample of at
    most 8 channels x 16 x 16 pixels per layer and, per sample, the sum and the sum of squares over the whole tensor;
  * ``forward`` images at truncation 1.0 and 0.37 (0.37 / 0.02 = 18.5: the statistics are interpolated) and for a list of 15
    distinct latents (one per layer), and BigGAN-128 images: each sub-sampled to 64^2 (every 8th / 2nd pixel), plus per-sample
    sums over the whole image.

Run:  python oracle/gen_golden_biggan_synth.py   (about half a minute of CPU time; the file is ~0.5 MB)
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
OUT = ROOT / "tests" / "golden" / "biggan_synthesis_known_answers.npz"
SEED = 4321
N = 2


def checksums(sd):
    keys = list(sd)
    sums = np.array([sd[k].double().sum().item() for k in keys])
    sq = np.array([sd[k].double().pow(2).sum().item() for k in keys])
    return np.array(keys), sums, sq


def subsample(t):
    """[n, C, R, R] -> [n, <=8, <=16, <=16] strided sub-sample."""
    c, r = t.shape[1], t.shape[2]
    return t[:, ::max(1, c // 8), ::max(1, r // 16), ::max(1, r // 16)].contiguous().numpy()


def main():
    from oracle import ref_harness
    from ganspace_b200.models.biggan import synthesis_fill
    ref = ref_harness.import_reference()
    dev = torch.device("cpu")
    torch.set_grad_enabled(False)
    out = {}

    m = ref_harness.rand_init_biggan512(ref, dev, "husky", SEED)
    synthesis_fill(m.model, SEED)
    m.eval()
    keys, sums, sq = checksums(m.model.state_dict())
    out.update(sd512_keys=keys, sd512_sum=sums, sd512_sq=sq,
               sd512_shapes=np.array([str(tuple(v.shape)) for v in m.model.state_dict().values()]))

    from models import biggan
    z = torch.from_numpy(biggan.truncated_noise_sample(truncation=1.0, batch_size=N, seed=11))
    z_list = [torch.from_numpy(biggan.truncated_noise_sample(truncation=1.0, batch_size=N, seed=100 + i))
              for i in range(m.model.n_latents)]
    out["z"] = z.numpy()
    out["z_list"] = np.stack([t.numpy() for t in z_list])

    acts = {}
    hooks = [layer.register_forward_hook(lambda mod, i, o, k=k: acts.__setitem__(k, o.detach().clone()))
             for k, layer in enumerate(m.model.generator.layers)]
    m.partial_forward(z, f"generator.layers.{len(m.model.generator.layers) - 1}")
    for h in hooks:
        h.remove()
    for k, a in sorted(acts.items()):
        out[f"act{k}_sub"] = subsample(a)
        out[f"act{k}_sum"] = a.double().sum(dim=(1, 2, 3)).numpy()
        out[f"act{k}_sq"] = a.double().pow(2).sum(dim=(1, 2, 3)).numpy()
        out[f"act{k}_shape"] = np.array(a.shape)
        out[f"act{k}_absmax"] = np.float64(a.abs().max())

    def image(tag, x):
        img = m.forward(x)
        out[f"img_{tag}_sub"] = img[:, :, ::8, ::8].contiguous().numpy()
        out[f"img_{tag}_sum"] = img.double().sum(dim=(1, 2, 3)).numpy()

    image("t100", z)
    m.truncation = 0.37
    z37 = torch.from_numpy(biggan.truncated_noise_sample(truncation=0.37, batch_size=N, seed=12))
    out["z37"] = z37.numpy()
    image("t037", z37)
    m.truncation = 1.0
    image("list", z_list)

    class RandInit128(ref.wrappers.BigGAN):
        def load_model(self, name):
            torch.manual_seed(SEED)
            self.model = biggan.BigGAN(biggan.BigGANConfig()).to(self.device)

    m128 = RandInit128(dev, 128, "husky")
    synthesis_fill(m128.model, SEED)
    m128.eval()
    keys, sums, sq = checksums(m128.model.state_dict())
    out.update(sd128_keys=keys, sd128_sum=sums, sd128_sq=sq)
    img = m128.forward(z)
    out["img128_sub"] = img[:, :, ::2, ::2].contiguous().numpy()
    out["img128_sum"] = img.double().sum(dim=(1, 2, 3)).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
