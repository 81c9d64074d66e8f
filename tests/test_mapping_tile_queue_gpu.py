"""The persistent layer kernel (mapping network, tc_linear, the synthesis tap GEMMs) hands out its tiles through a queue:
each CTA claims the next tile when it has room for it, so a CTA that starts late, its SM held by another stream's work,
takes fewer tiles.  Every tile goes through the same MMA sequence and epilogue, so results must not depend on which CTAs
start late."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def packed(mapping_weights):
    from ganspace_b200 import _native as nat
    nat.load()
    ws, bs = mapping_weights
    return nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)


@pytest.fixture(scope="module")
def z():
    return torch.randn((70_000, 512), generator=torch.Generator(device="cuda").manual_seed(11), device="cuda")


@pytest.mark.parametrize("free", [0, 32, 100])
@pytest.mark.parametrize("n", [1, 127, 128, 8193, 70_000])
def test_mapping_rows_independent_of_free_sms(packed, z, oracle, mapping_weights, n, free):
    full = packed.forward(z, leave_free_sms=0).cpu().numpy()
    out = packed.forward(z[:n], leave_free_sms=free).cpu().numpy()
    packed.check()
    assert np.array_equal(out, full[:n]), (n, free)
    ws, bs = mapping_weights
    ref = oracle.mapping_forward(z[n - min(n, 200):n].cpu().numpy(), ws, bs)
    assert np.max(np.abs(out[n - min(n, 200):] - ref)) < 2e-5 * np.max(np.abs(ref))


def _with_rng_on_side_stream(fn):
    """Runs fn() on the current stream right after an RNG launch group (56 CTAs, about a millisecond each) was queued on a
    side stream, so that some of fn's CTAs find their SMs taken and start late."""
    from ganspace_b200 import _native as nat
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    parts = nat.split_parts(512 * 10_000)
    with torch.cuda.stream(side):
        noise = nat.legacy_normal(list(range(7)), 512 * 10_000, torch.device("cuda:0"), parts=parts)
    out = fn()
    torch.cuda.current_stream().wait_stream(side)
    noise.record_stream(torch.cuda.current_stream())
    return out


@pytest.mark.parametrize("free", [0, 32])
def test_mapping_with_late_ctas(packed, z, free):
    ref = packed.forward(z, leave_free_sms=free).cpu().numpy()
    for _ in range(3):
        out = _with_rng_on_side_stream(lambda: packed.forward(z, leave_free_sms=free)).cpu().numpy()
        assert np.array_equal(out, ref), free
    packed.check()


def test_tensor_core_linear_with_late_ctas():
    """tc_linear (BigGAN gen_z's shape: [300, 256] x [32768, 256]^T) claims its tiles from a queue too."""
    from ganspace_b200 import _native as nat
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((300, 256), generator=g, device="cuda")
    w = torch.randn((32768, 256), generator=g, device="cuda") * 0.05
    b = torch.randn((32768,), generator=g, device="cuda")
    alone = nat.linear(x, w, b, bounded=True).cpu().numpy()
    shared = _with_rng_on_side_stream(lambda: nat.linear(x, w, b, bounded=True)).cpu().numpy()
    assert np.array_equal(alone, shared)
    ref = (x.double() @ w.double().T + b.double()).cpu().numpy()
    assert np.max(np.abs(alone - ref)) < 2e-5 * np.max(np.abs(ref))


def test_synthesis_tap_gemm_with_late_ctas(oracle):
    """tc_gemm_plain (the StyledConv tap GEMMs) claims its tiles from a queue too: the conv1 -> convs.0 -> convs.1 chain
    on two latents, alone and next to an RNG group, against the oracle."""
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    model.use_w()
    w = model.sample_latent(2, seed=7)
    inst = get_instrumented_model("StyleGAN2", "ffhq", "convs.1", dev, model=model, use_w=True)

    def run():
        model.partial_forward(w, "convs.1")
        return inst.retained_features()["convs.1"].clone()

    alone = run().cpu().numpy()
    shared = _with_rng_on_side_stream(run).cpu().numpy()
    assert np.array_equal(alone, shared)
    params = oracle.synthesis_random_init(1234, 1024, "convs.1")
    ref = oracle.synthesis_forward(w.cpu().numpy(), params, oracle.fixed_noise(0, 1024), "convs.1")
    assert np.abs(alone - ref).max() / np.abs(ref).max() < 2e-4
