"""ORACLE / TEST INFRASTRUCTURE -- StyleGAN (v1) style space: the StyleMod linears ``g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin``
(models/stylegan/model.py:121-136) restated on top of oracle/stylegan_oracle.py, whose functions are used unchanged:

  * ``style_rows``     the rows [n, 2C] = [s0 | s1] of one style layer, fp64
  * ``render_styled``  the image in the reference's form with every layer's style rows taken from the caller, any torch dtype

tests/test_stylegan_stylespace.py pins both to the unmodified reference (oracle/gen_golden_stylegan_stylespace.py).  Nothing
under ganspace_b200/ imports this module.
"""
import numpy as np

from oracle import stylegan_oracle as so


def style_layer_names(resolution):
    """The style layers ``g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin`` in execution order (chain layer l = entry l)."""
    return [f"{epi}.style_mod.lin" for _, _, epi, _, _ in so.layers({}, resolution)]


def style_rows(w, sd, epi):
    """The style-space rows [n, 2C] = [s0 | s1] of StyleMod ``epi``.style_mod.lin for dlatents w [n, 512] (fp64)."""
    return np.concatenate(so.style(w, sd, epi), axis=1)


def render_styled(S, sd, noise, resolution, dtype=None, device="cpu"):
    """The image 0.5 (torgb + 1) [n, 3, R, R] in the reference's form, with every layer's style rows taken from the caller:
    ``S`` {style layer name: rows [n, 2C]}; any torch dtype (default fp64) and device.  ``noise``: {res: [res, res] map}.
    Each layer is ``stylegan_oracle.layer_torch`` fed the rows as its dlatent through an identity StyleMod (weight
    sqrt(512) I, bias 0), which reproduces the rows exactly in any dtype."""
    import torch
    dtype = dtype or torch.float64
    T = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(so._np(a)))).to(device=device, dtype=dtype)
    sdt = {k: T(v) for k, v in sd.items() if k.startswith("g_synthesis.")}
    x = None
    for (_, conv, epi, up, r), name in zip(so.layers(sd, resolution), style_layer_names(resolution)):
        s = T(S[name])
        width = s.shape[1]
        lsd = dict(sdt)
        lsd[f"{epi}.style_mod.lin.weight"] = torch.eye(width, dtype=dtype, device=device) * float(np.sqrt(so.DLATENT))
        lsd[f"{epi}.style_mod.lin.bias"] = torch.zeros(width, dtype=dtype, device=device)
        x = so.layer_torch(x, s, lsd, conv, epi, up, T(noise[r]))
    W = sdt["g_synthesis.torgb.weight"][:, :, 0, 0]
    img = torch.einsum("bchw,oc->bohw", x, W / float(np.sqrt(W.shape[1]))) + sdt["g_synthesis.torgb.bias"].view(1, 3, 1, 1)
    return 0.5 * (img + 1)
