"""ORACLE -- BigGAN-deep conditional-BatchNorm rows in fp64 (pytorch_pretrained_biggan/model.py:99-149, wrappers.py:611-648).

Every GenBlock's four BatchNorms have a gain 1 + scale(cond) and a bias offset(cond), where scale and offset are bias-free
spectral-norm linears of the block's condition vector cond = [z, embed]:

    rows(generator.layers.k.bn_j.scale)  = cond W_eff^T,   W_eff = W_orig / sigma,   sigma = u^T W_orig v   (eval mode)

The weights are this repository's module tree under the reference's random init (``torch.manual_seed(seed)``, then
``synthesis_fill(net, seed)``), which test_biggan_synthesis.py checks against the reference's own checksums.
"""
import numpy as np
import torch

from oracle import ganspace_oracle as go

HUSKY = 248


def row_stride(c):
    """The channel stride of a layer's sub-sample in tests/golden/biggan_stylespace_known_answers.npz: at most 64 channels."""
    return max(1, c // 64)


def known_rows(ka, res, tag):
    """{name: (sub [n, <=64], sum [n], sum of squares [n])} of the reference's rows of every row layer of BigGAN-``res`` in
    biggan_stylespace_known_answers.npz, latent set ``tag`` ('z', or 'list' at 512); ``sub`` is rows[:, ::row_stride(C)]."""
    sub, sums, sq = ka[f"r{res}_{tag}_sub"], ka[f"r{res}_{tag}_sum"], ka[f"r{res}_{tag}_sq"]
    out, c0 = {}, 0
    for i, (name, c) in enumerate(zip(ka[f"r{res}_names"], ka[f"r{res}_widths"])):
        w = -(-int(c) // row_stride(int(c)))
        out[str(name)] = (sub[:, c0:c0 + w], sums[i], sq[i])
        c0 += w
    assert c0 == sub.shape[1]
    return out


def known_rows_err(rows, known):
    """Relative errors of full rows [n, C] against one ``known_rows`` entry: the sub-sample (max |diff| / max |known|), the
    per-sample sums of squares (max relative diff) and the per-sample sums (max |diff| / (C rms), C rms = sqrt(C sum of squares))."""
    sub, sums, sq = known
    rows = np.asarray(rows, np.float64)
    c = rows.shape[1]
    got_sub = rows[:, ::row_stride(c)]
    assert got_sub.shape == sub.shape, (got_sub.shape, sub.shape)
    return (float(np.abs(got_sub - sub).max() / np.abs(sub).max()),
            float(np.abs((rows ** 2).sum(1) - sq).max() / sq.max()),
            float(np.abs(rows.sum(1) - sums).max() / np.sqrt(c * sq.max())))


def net(resolution, seed=4321):
    from ganspace_b200.models import biggan
    torch.manual_seed(seed)
    m = biggan._BigGANNet(resolution)
    biggan.synthesis_fill(m, seed)
    return m


def weight64(m, name):
    """W_eff [C, 256] of row layer ``name`` in fp64."""
    lin = m.get_submodule(name)
    w = lin.weight_orig.detach().double()
    return w / torch.dot(lin.weight_u.double(), torch.mv(w, lin.weight_v.double()))


def embed64(m, class_idx=HUSKY):
    return m.embeddings.weight.detach().double()[:, class_idx]


def rows64(m, name, z, class_idx=HUSKY):
    """The rows [n, C] of row layer ``name`` for latents z [n, 128] in fp64 (numpy)."""
    z = torch.as_tensor(np.asarray(z)).double().reshape(-1, 128)
    cond = torch.cat((z, embed64(m, class_idx)[None].expand(z.shape[0], -1)), dim=1)
    return (cond @ weight64(m, name).T).numpy()


def compute_rows(m, name, n, B, c, class_idx=HUSKY, seed=None, ipca="svd"):
    """get_or_compute on row layer ``name`` in Z space, restated (decomposition.compute, ipca): latents from the reference's
    truncated-normal stream, activations the fp64 rows rounded to fp32 as the layer outputs them."""
    sample = lambda s, B_: go.truncated_noise_sample(s, B_)
    activate = lambda z: rows64(m, name, z, class_idx).astype(np.float32)
    return go.compute_path(sample, activate, 128, weight64(m, name).shape[0], n, B, c, False, seed=seed, ipca=ipca)
