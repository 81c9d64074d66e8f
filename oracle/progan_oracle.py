"""ORACLE / TEST INFRASTRUCTURE -- ProGAN generator (netdissect/proggan.py:34-171), restated twice:

  * ``progan_block_forward``  the reference's own form on the host (PixelNorm -> nearest x2 -> F.conv2d -> wscale -> leaky-ReLU)
  * ``progan_block_taps``     the form the kernels of csrc/progan.cu compute (fp64 NumPy): one contraction over ci per tap at the
                              INPUT resolution, then a gather -- tests/test_progan.py pins the two to each other
and ``progan_random_init``, the random weights ``ganspace_b200.models.progan.random_init`` and oracle/gen_golden_progan.py share.
Nothing under ganspace_b200/ imports this module.
"""
import numpy as np

SIZES_256 = [512, 512, 512, 512, 256, 128, 64, 32]


def block_specs(sizes=SIZES_256):
    """[(name, cin, cout, ksize, padding, upsample)] in execution order, output block last (proggan.py:72-87)."""
    specs = [("layer1", sizes[0], sizes[1], 4, 3, False), ("layer2", sizes[1], sizes[1], 3, 1, False)]
    for si, so in zip(sizes[1:-1], sizes[2:]):
        specs.append((f"layer{len(specs) + 1}", si, so, 3, 1, True))
        specs.append((f"layer{len(specs) + 1}", so, so, 3, 1, False))
    dim = 4 * 2 ** (len(specs) // 2 - 1)
    specs.append((f"output_{dim}x{dim}", sizes[-1], 3, 1, 0, False))
    return specs


def progan_random_init(seed=1234, sizes=SIZES_256):
    """{name: dict(weight [co,ci,k,k], b [co], ksize, upsample, scale)}: under torch.manual_seed(seed), per block in order a default
    nn.Conv2d init (consumed, as the reference's constructor does) and b ~ N(0,1); then every conv weight ~ N(0,1) in block order."""
    import torch
    torch.manual_seed(int(seed))
    params = {}
    for name, ci, co, k, pad, up in block_specs(sizes):
        torch.nn.Conv2d(ci, co, k, 1, pad, bias=False)
        gain = 1.0 if name.startswith("output") else np.sqrt(2) / k
        params[name] = dict(b=torch.randn(co).numpy(), ksize=k, padding=pad, upsample=up, scale=gain / np.sqrt(ci))
    for name, ci, co, k, pad, up in block_specs(sizes):
        params[name]["weight"] = torch.randn(co, ci, k, k).numpy()
    return params


def pixel_norm(x):
    """x / sqrt(mean_c x^2 + 1e-8) over axis 1 (NCHW)."""
    return x / np.sqrt(np.mean(x * x, axis=1, keepdims=True) + 1e-8)


def progan_block_forward(x, L, output=False, dtype=np.float32):
    """Reference form, torch on the host in ``dtype`` (float32: the reference's own arithmetic; float64: the per-layer parity
    reference of tests/test_progan_gpu.py).  x [B, ci, H, W] -> [B, co, H', W']."""
    import torch
    import torch.nn.functional as F
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=dtype))
    t = T(x)
    t = t / torch.sqrt(torch.mean(t ** 2, dim=1, keepdim=True) + 1e-8)
    if L["upsample"]:
        t = F.interpolate(t, scale_factor=2, mode="nearest")
    t = F.conv2d(t, T(L["weight"]), None, 1, L["padding"])
    t = t * float(L["scale"]) + T(L["b"]).view(1, -1, 1, 1)
    if not output:
        t = F.leaky_relu(t, 0.2)
    return t.numpy()


def progan_block_taps(x, L, output=False):
    """The kernels' form in fp64: Y[b,p,tap,co] at the input resolution, then the gather."""
    x = pixel_norm(np.asarray(x, np.float64))
    W = np.asarray(L["weight"], np.float64) * L["scale"]
    B, ci, H, _ = x.shape
    co, k = W.shape[0], L["ksize"]
    if k == 4:                                    # 1x1 latent, padding 3: output pixel (y, x) meets tap (3 - y, 3 - x)
        out = np.einsum("bc,ocyx->boyx", x[:, :, 0, 0], W[:, :, ::-1, ::-1])
    elif k == 1:
        out = np.einsum("bchw,oc->bohw", x, W[:, :, 0, 0])
    else:
        Y = np.einsum("bchw,ocyx->bhwyxo", x, W)                       # [B, H, H, 3, 3, co]
        R = 2 * H if L["upsample"] else H
        out = np.zeros((B, R, R, co))
        idx = np.arange(R)
        for ky in range(3):
            yy = idx + ky - 1
            my = (yy >= 0) & (yy < R)
            ys = (yy[my] >> 1) if L["upsample"] else yy[my]
            for kx in range(3):
                xx = idx + kx - 1
                mx = (xx >= 0) & (xx < R)
                xs = (xx[mx] >> 1) if L["upsample"] else xx[mx]
                out[np.ix_(np.arange(B), idx[my], idx[mx])] += Y[:, ys][:, :, xs][:, :, :, ky, kx, :]
        out = out.transpose(0, 3, 1, 2)
    out = out + np.asarray(L["b"], np.float64).reshape(1, -1, 1, 1)
    return out if output else np.where(out >= 0, out, 0.2 * out)


def progan_forward(z, params, upto=None, form="reference", keep=()):
    """Activation of block ``upto`` (default: the output block, i.e. the image before 0.5 (x + 1)) for z [B, 512]; with ``keep``
    (block names) returns {name: activation} instead."""
    fn = progan_block_forward if form == "reference" else progan_block_taps
    x = np.asarray(z).reshape(len(z), -1, 1, 1)
    kept = {}
    for name, L in params.items():
        x = fn(x, L, output=name.startswith("output"))
        if name in keep:
            kept[name] = x
        if name == upto:
            break
    return kept if keep else x
