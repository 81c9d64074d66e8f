"""Which activation edits the fused generator chains accept.  A forward hook that returns a new tensor edits its layer, and a
fused chain cannot take that tensor back: the edit raises when the run goes on past the edited layer, and is accepted on the
last layer of a partial run.  Each call path has its own rule:

| call path            | an edit raises when                                                                |
|----------------------|------------------------------------------------------------------------------------|
| StyleGAN2, StyleGAN  | the layer comes before the target, or when the image is made                       |
| ProGAN               | the layer comes before the target (the output block's result is the image         |
|                      | ``forward`` returns)                                                               |
| BigGAN               | before the last layer run, or when the image is made                               |
"""
from contextlib import contextmanager

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@contextmanager
def _hooked(*modules, edit=True):
    """Forward hooks on ``modules`` that edit (add 1) or only watch their layer."""
    hook = (lambda m, args, out: out + 1) if edit else (lambda m, args, out: None)
    handles = [m.register_forward_hook(hook) for m in modules]
    try:
        yield
    finally:
        for h in handles:
            h.remove()


def _raises():
    return pytest.raises(NotImplementedError, match="cannot be propagated")


def test_stylegan2_single_latent_partial_run():
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(DEV, "cat", random_init=3)
    z, g = m.sample_latent(2, seed=1), m.model
    with _hooked(g.convs[0]):
        m.partial_forward(z, "convs.0")
    with _hooked(g.conv1), _raises():
        m.partial_forward(z, "convs.0")


def test_stylegan2_per_layer_path():
    """Per-layer latents, or a ToRGB hooked on the way: every ToRGB such a run executes comes before the target, so an edit of
    the target is accepted; the ToRGB's own edit and that of the StyledConv a ToRGB target follows raise."""
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(DEV, "cat", random_init=3)
    z, g = m.sample_latent(2, seed=1), m.model
    with _hooked(g.to_rgb1, edit=False), _hooked(g.convs[0]):
        m.partial_forward(z, "convs.0")
    with _hooked(g.convs[0]):
        m.partial_forward([z, z], "convs.0")
    with _hooked(g.to_rgbs[0]):
        m.partial_forward([z, z], "to_rgbs.0")
    with _hooked(g.to_rgb1), _raises():
        m.partial_forward(z, "convs.0")
    with _hooked(g.convs[1]), _raises():
        m.partial_forward([z, z], "to_rgbs.0")
    with _hooked(g.conv1), _raises():
        m.partial_forward([z, z], "convs.0")
    with _hooked(g.to_rgbs[0]), _raises():
        m.forward(z)


def test_progan():
    from ganspace_b200.models import ProGAN
    m = ProGAN(DEV, "bedroom", random_init=3)
    z, g = m.sample_latent(2, seed=1), m.model
    with _hooked(g.layer3):
        m.partial_forward(z, "layer3")
    with _hooked(g.layer2), _raises():
        m.partial_forward(z, "layer3")
    plain = m.forward(z)
    with _hooked(g._modules[g.block_names()[-1]]):
        edited = m.forward(z)
    assert torch.allclose(edited, plain + 0.5, atol=1e-6)


def test_stylegan():
    from ganspace_b200.models import StyleGAN
    m = StyleGAN(DEV, "bedrooms", random_init=3)
    z, blocks = m.sample_latent(2, seed=1), m.model.g_synthesis.blocks
    with _hooked(blocks["8x8"]):
        m.partial_forward(z, "g_synthesis.blocks.8x8")
    with _hooked(blocks["4x4"]), _raises():
        m.partial_forward(z, "g_synthesis.blocks.8x8")
    with _hooked(blocks["256x256"]), _raises():
        m.forward(z)


def test_biggan():
    from ganspace_b200.models.biggan import BigGAN
    m = BigGAN(DEV, 128, "husky", random_init=3)
    z, layers = m.sample_latent(2, seed=1), m.model.generator.layers
    with _hooked(layers[3]):
        m.partial_forward(z, "generator.layers.3")
    with _hooked(layers[2]), _raises():
        m.partial_forward(z, "generator.layers.3")
    with _hooked(layers[len(layers) - 1]), _raises():
        m.forward(z)
