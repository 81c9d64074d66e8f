"""Decomposition driver: ``get_or_compute`` / ``compute`` -- the hot path's public entry point.

Mirror of /root/reference/decomposition.py (get_or_compute :362-368, _compute :370-402, compute :150-358,
linreg_lstsq :77-139, get_random_dirs :42-46, get_max_batch_size :49-74): same signature, validation
errors, cache-file naming, seeding protocol and 8-array ``.npz`` schema, so ``visualize.py``,
``interactive.py`` and the notebooks consume the result unchanged.

What changed is where the work happens.  The reference samples latents on the host, round-trips every
batch through host memory and runs sklearn's IncrementalPCA on the CPU; here
  * every NumPy-legacy latent stream of the run is generated on the GPU (one CTA per sample_latent seed),
  * the mapping network / hooked layer runs in hand-written CUDA kernels,
  * the IncrementalPCA merge chain runs on the device from per-group (mean, centred Gram) statistics,
  * the regression pass accumulates normal equations on the device,
so activations never leave HBM; the host only draws the seeds (NumPy global state, as the reference
does) and receives the final components.

Multi-GPU (one process per GPU, torch.distributed initialised): partial_fit group k belongs to rank k mod world; the run
proceeds in rounds of world x g groups: every rank computes the statistics of its g groups, one all-gather per round hands
them to every rank, and every rank merges them into its replica of the chain in the reference's order while the next round
is already being computed -- the result does not depend on the world size (SURVEY.md section 8e).
"""
from __future__ import annotations

import copy
import datetime
import inspect
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

from . import _native
from . import plan as _plan
from .config import Config  # noqa: F401  (re-exported like the reference module does)
from .estimators import DeviceIncrementalPCA, get_estimator
from .models import get_instrumented_model
from .netdissect.nethook import InstrumentedModel

SEED_SAMPLING = 1
SEED_RANDOM_DIRS = 2
SEED_LINREG = 3
SEED_VISUALIZATION = 5

B = 20
n_clusters = 500

# bytes of latents generated per pipeline chunk (8 GiB of the 80 GB HBM keeps config 2 in one chunk)
LATENT_CHUNK_BYTES = 8 << 30
# partial_fit groups whose statistics are computed by one set of launches (the first block is small so that the merge
# chain starts early; 10 groups x 10 tile pairs at d = 512 are 100 work items, one wave on the 132 SMs)
STATS_FIRST_BLOCK = int(os.environ.get("GANSPACE_B200_STATS_FIRST", 4))
STATS_BLOCK = int(os.environ.get("GANSPACE_B200_STATS_BLOCK", 10))


def get_random_dirs(components, dimensions):
    gen = np.random.RandomState(seed=SEED_RANDOM_DIRS)
    dirs = gen.normal(size=(components, dimensions))
    dirs /= np.sqrt(np.sum(dirs ** 2, axis=1, keepdims=True))
    return dirs.astype(np.float32)


def get_max_batch_size(inst, device, layer_name=None):
    """Largest probe batch (<= 20) whose peak memory stays under half the device (reference :49-74)."""
    inst.remove_edits()
    torch.cuda.reset_peak_memory_stats(device)
    total_mem = torch.cuda.get_device_properties(device).total_memory
    B_max = 20
    for i in range(2, B_max, 2):
        z = inst.model.sample_latent(n_samples=i)
        if layer_name:
            inst.model.partial_forward(z, layer_name)
        else:
            inst.model.forward(z)
        maxmem = torch.cuda.max_memory_allocated(device)
        del z
        if maxmem > 0.5 * total_mem:
            print("Batch size {:d}: memory usage {:.0f}MB".format(i, maxmem / 1e6))
            return i
    return B_max


def _dist():
    """(rank, world, group-is-live) of the data-parallel job, (0, 1, False) when not distributed."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_rank(), dist.get_world_size(), True
    return 0, 1, False


class _StatsExchange:
    """All-gather of one round's per-group statistics (SURVEY.md section 8e; plan.rounds).  ``start`` enqueues the
    collective asynchronously; ``finish`` (called one round later, so that the next round's kernels are already queued behind
    it) merges the round's groups into this rank's chain replica in the reference's group order."""

    def __init__(self, d, world):
        self.d, self.world = d, world

    def start(self, rnd, means, grams):
        import torch.distributed as dist
        g = means.shape[0]
        recv_m = torch.empty((self.world * g, self.d), dtype=torch.float64, device=means.device)
        recv_g = torch.empty((self.world * g, self.d, self.d), dtype=torch.float64, device=means.device)
        works = [dist.all_gather_into_tensor(recv_g, grams, async_op=True),
                 dist.all_gather_into_tensor(recv_m, means, async_op=True)]
        return rnd, g, recv_m, recv_g, works, (means, grams)          # the send buffers stay alive until finish()

    def finish(self, pending, transformer, NB):
        rnd, g, recv_m, recv_g, works, _keep = pending
        for w in works:
            w.wait()
        for kk in rnd:
            slot = (kk % self.world) * g + (kk - rnd[0]) // self.world
            if not transformer.fit_partial_stats(NB, recv_m[slot], recv_g[slot]):
                return False
        return True


def _draw_seeds(count):
    """``count`` successive ``np.random.randint(int32 max)`` draws on the global state, i.e. the seeds that
    ``count`` successive ``sample_latent()`` calls would consume (models/wrappers.py:168-169)."""
    hi = np.iinfo(np.int32).max
    return [int(np.random.randint(hi)) for _ in range(count)]


def _sample_batches(model, Bsz, seeds, out=None):
    """Rows of len(seeds) consecutive ``sample_latent(Bsz)`` calls, as one [len*Bsz, ...] device tensor."""
    if hasattr(model, "sample_latents_multi"):
        return model.sample_latents_multi(Bsz, seeds, out=out)
    return torch.cat([model.sample_latent(Bsz, seed=s) for s in seeds], dim=0)


def _sample_batches_lazy(model, Bsz, seeds):
    """Like _sample_batches, plus ``ensure(row_end)``: rows [0, row_end) are final once it returns.  Models whose
    sample_latent has a second stage (StyleGAN2 W space: the mapping network) run it chunk by chunk on demand,
    so the IPCA chain starts on the first groups while later rows are still being mapped."""
    fn = getattr(model, "sample_latents_multi", None)
    if fn is not None and "lazy" in inspect.signature(fn).parameters:
        return fn(Bsz, seeds, lazy=True)
    return _sample_batches(model, Bsz, seeds), (lambda row_end: None)


# Solve for directions in latent space that match PCs in activation space (reference :77-139)
def linreg_lstsq(comp_np, mean_np, stdev_np, inst, config, affine=None, native=False, act_buf=None):
    """``affine``: when the hooked layer is affine in the latent (models/biggan.py AffineLayer), comp/mean are
    given in its r-dimensional coordinates and the projections run there: (act-mean).comp^T == (y-ybar).comp_y^T.
    ``native``: comp/mean are given in the model's device feature order (``feature_layout``) and the activations
    come from ``model.activations_into`` in that same order (no hook read-back, no permutation); comp/mean may then be
    device tensors.  ``act_buf``: [>= B, d] rows the native producer may overwrite (the large-d engine's batch rows, once
    nothing reads them), instead of a new [B, d] buffer."""
    print("Performing least squares regression", flush=True)
    torch.manual_seed(SEED_LINREG)
    np.random.seed(SEED_LINREG)
    model = inst.model
    dev = model.device
    # comp / mean may be device tensors already (conv layers: the engine's export in the device feature order)
    as_dev = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(a)).float().to(dev)
    comp = as_dev(comp_np).contiguous()
    mean = as_dev(mean_np).reshape(-1).contiguous()
    stdev = torch.from_numpy(stdev_np).float().to(dev).contiguous()

    n_samp = max(10_000, config.n) // B * B
    n_comp = comp.shape[0]
    latent_dims = int(model.get_latent_dims())      # consumes one global draw, as in the reference (:88)
    rank, world, live = _dist()

    acc = _native.LinregAccumulator(n_comp, latent_dims, dev)
    if native and act_buf is None:
        act_buf = torch.empty((B, comp.shape[1]), dtype=torch.float32, device=dev)
    elif native:
        act_buf = act_buf[:B]
    seeds = _draw_seeds(n_samp // B)
    group = max(1, min(len(seeds), (256 << 20) // max(1, B * latent_dims * 4)))
    for start in range(0, len(seeds), group):
        idx = [i for i in range(start, min(start + group, len(seeds))) if i % world == rank]
        if not idx:
            continue
        z_all = _sample_batches(model, B, [seeds[i] for i in idx])
        for j in range(len(idx)):
            z = z_all[j * B:(j + 1) * B]
            if affine is not None:
                act = affine.coords(z.reshape(B, -1))
            elif native:
                act = model.activations_into(z, config.layer, act_buf)
            else:
                with torch.no_grad():
                    model.partial_forward(z, config.layer)
                act = inst.retained_features()[config.layer].reshape(B, -1)
            acc.accumulate(act.contiguous(), comp, mean, stdev, z.reshape(B, -1).contiguous())
    if live:
        import torch.distributed as dist
        flat = acc.state.view(torch.float64)
        dist.all_reduce(flat)
    acc.n_total = n_samp
    M_t, Z_mean = acc.solve()
    return M_t.cpu().numpy()[:n_comp, :], Z_mean.cpu().numpy().reshape(1, -1)


def _warn_if_not_orthonormal(comp):
    M = np.dot(comp, comp.T)
    # fp32 components (large-d engine) are orthonormal to ~1e-6, the reference's float64 ones to 1e-15
    if not np.allclose(M, np.identity(M.shape[0]), atol=1e-8 if comp.dtype == np.float64 else 5e-6):
        det = np.linalg.det(M)
        print(f"WARNING: Computed basis is not orthonormal (determinant={det})")


def regression(comp, mean, stdev, inst, config, affine=None, native=False, act_buf=None, host_comp=None):
    """``host_comp``: a host copy of ``comp`` (any feature order) for the orthonormality check when ``comp`` is a device tensor."""
    _warn_if_not_orthonormal(comp if host_comp is None else host_comp)
    return linreg_lstsq(comp, mean, stdev, inst, config, affine=affine, native=native, act_buf=act_buf)


def compute(config, dump_name, instrumented_model):
    """decomposition.compute (:150-358): run the pipeline, rank 0 writes the 8-array .npz."""
    timestamp = lambda: datetime.datetime.now().strftime("%d.%m %H:%M")
    print(f"[{timestamp()}] Computing", dump_name.name)
    state = {}
    try:
        arrays = compute_arrays(config, instrumented_model, state)
    except _native.ChainNotConverged as err:
        # the iterated chain step found no spectral gap after component c (e.g. activations of numerical rank < n_components):
        # run again with sklearn's own exact per-step eigen-solve (every rank of a distributed run sees the same status)
        print(f"{err}\nRe-running with the direct chain step", flush=True)
        _native.set_chain_mode(True)
        try:
            state = {}
            arrays = compute_arrays(config, instrumented_model, state)
        finally:
            _native.set_chain_mode(False)
    if state.get("canceled_at") is not None:
        # Ctrl-C during the fitting loop: the reference saves what was fitted so far under n{gi} and exits 1 (:268-274,342-343)
        dump_name = dump_name.parent / dump_name.name.replace(f"n{state['N']}", f"n{state['canceled_at']}")
        print(f'Saving current state to "{dump_name.name}" before exiting')
    rank, world, live = _dist()
    if rank == 0:
        _write_npz(dump_name, arrays)
    if live:
        import torch.distributed as dist
        dist.barrier()
    if state.get("canceled_at") is not None:
        sys.exit(1)


def _write_npz(dump_name, arrays):
    os.makedirs(dump_name.parent, exist_ok=True)
    # same 8-array .npz container, read by np.load exactly like the reference's; stored WITHOUT deflate: the arrays are
    # float32 noise (7 % smaller compressed) and single-core zlib costs 8-18 ms for config 2 -- a fifth of the whole
    # device run -- and minutes for conv feature maps (act_comp = 168 MB at convs.4).  GANSPACE_B200_NPZ_COMPRESS=1 restores
    # np.savez_compressed (decomposition.py:331-341).
    compress = os.environ.get("GANSPACE_B200_NPZ_COMPRESS") == "1" and sum(a.nbytes for a in arrays.values()) <= (64 << 20)
    (np.savez_compressed if compress else np.savez)(dump_name, **arrays)


def _phase_timer():
    """GANSPACE_B200_TIMING=1: print wall-clock per phase (synchronising); otherwise a no-op."""
    if os.environ.get("GANSPACE_B200_TIMING") != "1":
        return lambda label: None
    import time
    state = {"t": time.perf_counter()}

    def tick(label):
        torch.cuda.synchronize()
        now = time.perf_counter()
        print(f"[timing] {label}: {now - state['t']:.3f} s", flush=True)
        state["t"] = now
    return tick


def _export_components(transformer, affine, pooled, sample_dims, device):
    """The fitted estimator's result in the layer's coordinates: (X_comp, X_stdev, X_var_ratio, device mean, X_global_mean) for
    the file, and (Y_comp, Y_mean) for the regression (an affine layer's r-dimensional coordinates)."""
    tr = transformer.transformer
    X_comp, X_stdev, X_var_ratio = transformer.get_components()
    X_comp = np.array(X_comp, copy=True)
    mean_dev = transformer.device_outputs["mean"] if pooled else tr.device_attributes()["mean"]
    if affine is None:
        X_global_mean = (transformer.pooled_mean if pooled else tr.mean_).reshape((1, sample_dims))
        Y_comp, Y_mean = X_comp, X_global_mean              # device feature order (== the reference's unless `layout`)
    else:
        # lift through the isometry: components = components_y Q^T (svd_flip's sign rule is applied on the lifted
        # rows, as sklearn would on the full activations), mean = mean_y Q^T + offset
        lifted = affine.lift_rows(torch.from_numpy(X_comp).to(device))
        idx = torch.argmax(lifted.abs(), dim=1)
        signs = torch.sign(lifted[torch.arange(lifted.shape[0], device=device), idx])
        Y_comp = X_comp * signs.cpu().numpy()[:, None]
        Y_mean = (transformer.pooled_mean if pooled else tr.mean_).reshape((1, affine.Q.shape[1]))
        X_comp = (lifted * signs[:, None]).cpu().numpy()
        X_global_mean = (affine.lift_rows(mean_dev[None, :]) + affine.offset[None, :]).cpu().numpy()
    return X_comp, X_stdev, X_var_ratio, mean_dev, X_global_mean, Y_comp, Y_mean


def _final_arrays(config, X_comp, X_global_mean, X_stdev, X_var_ratio, Z_comp, Z_global_mean, rand_std_dev, lat_samples,
                  sample_shape, input_shape, input_dims, to_nchw):
    """The 8 arrays of the file from the exported result: the reference's shapes, and lat_stdev (W space: the spread of 5000
    latents, ``lat_samples()``, along the latent components) read back together with random_stdevs."""
    X_comp = to_nchw(X_comp).reshape(-1, *sample_shape)
    X_global_mean = to_nchw(X_global_mean).reshape(sample_shape)
    Z_comp = Z_comp.reshape(-1, *input_shape)
    Z_global_mean = Z_global_mean.reshape(input_shape)

    lat_stdev = np.ones_like(X_stdev)
    if config.use_w:
        samples = lat_samples()
        zc = torch.from_numpy(Z_comp.reshape(-1, input_dims).astype(np.float32))
        both = torch.cat([rand_std_dev.reshape(-1), _native.project_std(samples.contiguous(), zc).reshape(-1)]).cpu().numpy()
        X_stdev_random, lat_stdev = both[:rand_std_dev.numel()], both[rand_std_dev.numel():]
    else:
        X_stdev_random = rand_std_dev.cpu().numpy()
    return {
        "act_comp": X_comp.astype(np.float32),
        "act_mean": X_global_mean.astype(np.float32),
        "act_stdev": X_stdev.astype(np.float32),
        "lat_comp": Z_comp.astype(np.float32),
        "lat_mean": Z_global_mean.astype(np.float32),
        "lat_stdev": lat_stdev.astype(np.float32),
        "var_ratio": X_var_ratio.astype(np.float32),
        "random_stdevs": X_stdev_random.astype(np.float32),
    }


def compute_arrays(config, instrumented_model, state=None):
    """Everything of compute() up to (not including) the file write; returns the 8 float32 arrays.
    ``state`` (optional dict) receives N and, after a KeyboardInterrupt in the fitting loop, ``canceled_at`` = the
    number of samples fitted so far (single-process runs; the result then describes that prefix of the chain)."""
    global B
    tick = _phase_timer()
    state = {} if state is None else state

    torch.manual_seed(0)
    np.random.seed(0)

    device = _native.require_cuda("cuda")      # no CPU fallback (the reference falls back to 'cpu', :163-164)
    rank, world, live = _dist()
    layer_key = config.layer

    if instrumented_model is None:
        inst = get_instrumented_model(config.model, config.output_class, layer_key,
                                      torch.device("cuda", torch.cuda.current_device()))
        model = inst.model
    else:
        print("Reusing InstrumentedModel instance")
        inst = instrumented_model
        model = inst.model
        inst.remove_edits()
        model.set_output_class(config.output_class)
    device = model.device

    if config.use_w:
        print("Using W latent space")
        model.use_w()

    inst.retain_layer(layer_key)
    model.partial_forward(model.sample_latent(1), layer_key)
    sample_shape = inst.retained_features()[layer_key].shape
    sample_dims = int(np.prod(sample_shape))
    print("Feature shape:", sample_shape)

    input_shape = inst.model.get_latent_shape()
    input_dims = int(inst.model.get_latent_dims())

    config.components = min(config.components, sample_dims)
    # layers that are affine in the latent expose a thin factorisation act = (z R^T) Q^T + offset; the PCA then
    # runs on the r-dimensional coordinates and is lifted through the isometry Q at the end (models/biggan.py)
    affine = model.affine_layer(layer_key) if hasattr(model, "affine_layer") else None
    if affine is not None and config.components > affine.rank:
        raise NotImplementedError(f"components={config.components} exceeds the rank {affine.rank} of layer {layer_key}")
    transformer = get_estimator(config.estimator, config.components, config.sparsity, device=device)
    tr = transformer.transformer
    # fbpca (the one non-batched estimator on the device path) pools the per-group statistics instead of merging them into a
    # chain, and solves once at the end (estimators.FacebookPCAEstimator, csrc/rsvd.cu)
    pooled = not transformer.batch_support
    samples_are_latents = layer_key in ["g_mapping", "style"] and inst.model.latent_space_name() == "W"
    if pooled and affine is not None:
        # fbpca decomposes the stacked sample matrix, whose unfilled tail rows are zero activations, outside the affine image:
        # in the layer's linear form act = yt Qt^T (Qt: Q and the offset's direction) they are zero coordinates, so the pool
        # of coordinate statistics is the stacked matrix's (DESIGN.md section 5g)
        affine = affine.linear_form()
    # conv feature maps (d up to ~10^6): the large-d IPCA engine keeps sklearn's stacked matrix in HBM and the model's
    # producer kernels write each batch into it in the device feature order (NHWC); the fixed NHWC->NCHW permutation
    # is applied once to the exported components (PCA is equivariant under it)
    small_d_max = transformer.SMALL_D_MAX if pooled else transformer.transformer.SMALL_D_MAX
    large_d = affine is None and not samples_are_latents and sample_dims > small_d_max
    if pooled and large_d:
        raise NotImplementedError(f"--est {config.estimator} is not available for conv feature maps (d = {sample_dims} > "
                                  f"{small_d_max}); use --est ipca")
    layout = model.feature_layout(layer_key) if (large_d and hasattr(model, "feature_layout")) else None
    if large_d and live:
        # row-parallel generation + feature-sharded chain (SURVEY.md section 8e): rank r synthesises rows
        # [r NB/W, (r+1) NB/W) of every group, one all-to-all hands rank r the feature block r of all NB rows, the
        # small-side Gram is all-reduced, every rank solves the same small eigenproblem and updates its block.
        if layout is None:
            raise NotImplementedError("feature-sharded large-d runs need a model with activations_into / feature_layout")
        transformer.transformer.enable_feature_sharding(rank, world)
    if layout is not None:
        lh, lw, lc = layout[1]
        to_nchw = lambda A: np.ascontiguousarray(A.reshape(A.shape[0], lh, lw, lc).transpose(0, 3, 1, 2)).reshape(A.shape[0], -1)
        to_native = lambda A: np.ascontiguousarray(A.reshape(A.shape[0], lc, lh, lw).transpose(0, 2, 3, 1)).reshape(A.shape[0], -1)
    else:
        to_nchw = to_native = lambda A: A

    B = config.batch_size or get_max_batch_size(inst, device, layer_key)
    pl = _plan.make_plan(config.n, B, config.components)
    N, NB = pl.N, pl.NB
    print("B={}, N={}, dims={}, N/dims={:.1f}".format(B, N, sample_dims, N / sample_dims), flush=True)
    # conv feature maps whose components are large enough to matter (c d >= 4 M) are read back already permuted to NCHW: one
    # device transpose and one copy, instead of a host copy in NHWC plus a permuted host copy
    device_layout = layout is not None and config.components * sample_dims >= (1 << 22)
    if large_d and layout is not None and hasattr(model, "activations_workspace_bytes"):
        # the engine's stacked matrix and its producer's scratch have to fit the device together: check before anything runs
        reserve = model.activations_workspace_bytes(layer_key, B)
        need = _native.BigIPCA.device_bytes(sample_dims // world if live else sample_dims, config.components, NB)
        _native.check_device_memory(need + reserve, device, f"{model.model_name} {layer_key} (d = {sample_dims}, "
                                    f"{config.components} components, batches of {NB}): the large-d IPCA engine "
                                    f"({need:,} bytes) and the synthesis workspace ({reserve:,} bytes)")
    if device_layout:
        tr.host_layout = (layout[1][0] * layout[1][1], layout[1][2])

    torch.manual_seed(config.seed or SEED_SAMPLING)
    np.random.seed(config.seed or SEED_SAMPLING)

    # ---- Phase A: the seeds of every sample_latent(B) call the reference makes (:232-236) ----------
    seeds = _draw_seeds(pl.n_calls)
    # fbpca draws its test matrix from the global state when it fits, after the collection (:284) and before the W-space
    # lat_stdev seed (:327); nothing in between draws, so it is the next draw here
    if pooled and affine is not None and transformer.l >= affine.rank:
        # fbpca's range covers every direction of the rank-deficient samples: its exact branch, which needs no test matrix.
        # The reference still draws one here, but the next reader of the global state is the regression pass, which re-seeds
        # it first (np.random.seed(SEED_LINREG), decomposition.py:81), so skipping the draw changes no later draw.
        omega = None
    elif pooled and affine is not None and transformer.randomized(N + NB, sample_dims) and N + NB < sample_dims:
        raise NotImplementedError(f"--est {config.estimator} on layer {layer_key} with l = {transformer.l} < rank "
                                  f"{affine.rank} needs N + NB >= {sample_dims} samples (with fewer, fbpca draws its test "
                                  "matrix over the samples); use more samples, more components or --est ipca")
    else:
        omega = transformer.draw_omega(N + NB, sample_dims) if pooled else None
    # W-space runs end with model.sample_latent(5000) for lat_stdev (:325-329).  Without a regression pass nothing touches the
    # global NumPy state in between, so its seed is the next draw; its latent stream (one sequential MT19937 stream, ~6 ms on
    # one SM) is generated on a side stream while the run proceeds instead of at the tail of the critical path.
    lat_stdev_z = None
    if config.use_w and samples_are_latents and hasattr(model, "draw_z_async"):
        lat_stdev_z = model.draw_z_async(5000, _draw_seeds(1)[0])

    # ---- Phase B: per-group statistics + merge chain (:239-265) ------------------------------------
    K = pl.K
    d = affine.Q.shape[1] if affine is not None else sample_dims
    groups_per_chunk = max(1, int(LATENT_CHUNK_BYTES // max(1, NB * input_dims * 4)))
    X = None
    state["N"] = N
    k = 0
    stop = False                 # fit_partial returned False (e.g. n_components > first batch): the reference leaves the loop (:262-263)
    exchange = _StatsExchange(d, world) if (live and not large_d) else None
    # fbpca's random_stdevs project the first rows of the whole sample matrix (:313-316): rows [0, K NB) hold group data, the
    # rest of the first min(5000, N + NB) rows stay zero.  Each row is written by the rank that owns its group.
    first = torch.zeros((min(5000, N + NB), d), dtype=torch.float32, device=device) if pooled else None

    def group_rows(rows):
        """[n, d] activations of the hooked layer for latent rows ``rows`` (small-d engine; n is a multiple of NB)."""
        if samples_are_latents:
            return rows
        if affine is not None:
            return affine.coords(rows)
        out = torch.empty((rows.shape[0], d), dtype=torch.float32, device=device)
        for g0 in range(0, rows.shape[0], NB):
            for mb in range(0, NB, B):
                z = rows[g0 + mb:g0 + mb + B].reshape(-1, *input_shape[1:])
                with torch.no_grad():
                    model.partial_forward(z, layer_key)
                batch = inst.retained_features()[layer_key].reshape((z.shape[0], -1))
                space_left = min(B, NB - mb)
                out[g0 + mb:g0 + mb + space_left] = batch[:space_left]
        return out

    try:
        for c0 in range(0, K, groups_per_chunk):
            if stop:
                break
            c1 = min(c0 + groups_per_chunk, K)
            if large_d:                              # every rank takes part in every group (its row range)
                mine = list(range(c0, c1))
            else:
                mine = _plan.groups_to_process(pl, rank, world, c0, c1)
            runs = _plan.contiguous_runs(mine)
            # every sample_latent call this rank needs for the chunk, generated by ONE launch (one CTA per seed)
            needed, offsets = _plan.batch_slots(pl, runs)
            lat, ensure_rows = _sample_batches_lazy(model, B, [seeds[b] for b in needed])
            lat = lat.reshape(lat.shape[0], -1)
            if large_d:
                for run, off in zip(runs, offsets):
                    if stop:
                        break
                    for k in run:
                        r = off + (k - run[0]) * NB
                        ensure_rows(r + NB)
                        rows = lat[r:r + NB]
                        X = tr.batch_buffer(NB, d, device)              # rows of the engine's stacked matrix, in HBM
                        lo, hi = (rank * (NB // world), (rank + 1) * (NB // world)) if live else (0, NB)   # this rank's rows
                        for mb in range(0, NB, B):
                            a, b_ = max(mb, lo), min(mb + min(B, NB - mb), hi)
                            if a >= b_:
                                continue
                            z = rows[a:b_].reshape(-1, *input_shape[1:])
                            if layout is not None:
                                model.activations_into(z, layer_key, X[a - lo:b_ - lo])
                            else:
                                with torch.no_grad():
                                    model.partial_forward(z, layer_key)
                                X[a - lo:b_ - lo] = inst.retained_features()[layer_key].reshape((z.shape[0], -1))
                        if not transformer.fit_partial_inplace(NB):
                            stop = True
                            break
            else:
                # small-d engine: rounds of world x g consecutive groups.  The statistics (mean, centred Gram) of this rank's
                # g groups of a round come out of one set of launches (tensor-core Gram, csrc/stats_tc.cu); the chain steps
                # follow in the reference's group order, on every rank, from the all-gathered statistics.
                where = {kk: off + (kk - run[0]) * NB for run, off in zip(runs, offsets) for kk in run}
                pending = None
                for rnd in _plan.rounds(c0, c1, world, STATS_FIRST_BLOCK if c0 == 0 else STATS_BLOCK, STATS_BLOCK):
                    if stop:
                        break
                    own = [kk for kk in rnd if _plan.owner(kk, world) == rank]
                    g_max = -(-len(rnd) // world)
                    means = torch.zeros((g_max, d), dtype=torch.float64, device=device)
                    grams = torch.zeros((g_max, d, d), dtype=torch.float64, device=device) if (live and len(own) < g_max) \
                        else torch.empty((g_max, d, d), dtype=torch.float64, device=device)
                    if own:
                        k = own[0]
                        contiguous = all(where[own[i]] == where[own[0]] + i * NB for i in range(len(own)))
                        spans = [own] if contiguous else [[kk] for kk in own]
                        i0 = 0
                        for span in spans:
                            r0 = where[span[0]]
                            ensure_rows(r0 + len(span) * NB)
                            Xb = group_rows(lat[r0:r0 + len(span) * NB])
                            _native.batch_stats_multi(Xb, len(span), NB, mean_out=means[i0:i0 + len(span)],
                                                      gram_out=grams[i0:i0 + len(span)])
                            i0 += len(span)
                            if first is not None and span[0] * NB < first.shape[0]:
                                cnt = min(first.shape[0] - span[0] * NB, len(span) * NB)
                                first[span[0] * NB:span[0] * NB + cnt] = Xb[:cnt]
                        X = Xb[(len(span) - 1) * NB:]
                    if (K - 1) in rnd and _plan.owner(K - 1, world) != rank:
                        r0 = where[K - 1]                                # every rank keeps the final group's sample buffer
                        ensure_rows(r0 + NB)
                        X = group_rows(lat[r0:r0 + NB])
                    if exchange is None:
                        for i, kk in enumerate(own):
                            k = kk
                            if not transformer.fit_partial_stats(NB, means[i], grams[i]):
                                stop = True
                                break
                    else:
                        cur = exchange.start(rnd, means, grams)
                        if pending is not None and not exchange.finish(pending, transformer, NB):
                            stop = True
                        pending = cur
                        if rnd[0] < 2 * world * STATS_BLOCK and not stop:
                            # the first rounds are merged at once (the chain is idle and waiting for them); later rounds one
                            # round late, so that the collective overlaps the next round's kernels
                            if not exchange.finish(pending, transformer, NB):
                                stop = True
                            pending = None
                if pending is not None and not stop and not exchange.finish(pending, transformer, NB):
                    stop = True
            ensure_rows(lat.shape[0])
            del lat    # X (a view of the last group when samples_are_latents) keeps its storage alive
    except KeyboardInterrupt:
        if live:
            raise
        if pooled:
            sys.exit(1)          # nothing fitted yet, and the reference writes nothing (:269-270)
        # the reference's `gi` of the interrupted group (:268-272) = the samples merged so far
        state["canceled_at"] = int(tr.n_samples_seen_)
    if pooled:
        if live:
            import torch.distributed as dist
            dist.all_reduce(first)                               # each row is non-zero on exactly one rank
        transformer.add_zero_rows(N + NB - K * NB)               # the unfilled tail of the sample matrix (:224)
        if affine is not None:
            transformer.fit_pooled_affine(omega, affine.Q, affine.rank)
        else:
            transformer.fit_pooled(omega=omega)
    tick("sampling + activations + IPCA chain")
    # host work that does not depend on the chain's result, done while the device still runs the last merge steps (the
    # export below is the first call that waits for them): get_random_dirs' host stream + upload, the lat_stdev latents
    device_dirs = device_layout
    pre_dirs = None if device_dirs else \
        torch.from_numpy(to_native(get_random_dirs(config.components, int(np.prod(sample_shape))))).to(device, non_blocking=True)
    pre_lat = model.z_to_latent(lat_stdev_z()).reshape(5000, input_dims) if (config.use_w and lat_stdev_z is not None) else None
    X_comp, X_stdev, X_var_ratio, mean_dev, X_global_mean, Y_comp, Y_mean = \
        _export_components(transformer, affine, pooled, sample_dims, device)
    host_comp = None
    if device_layout:
        # X_comp / X_global_mean came back in NCHW order; the regression runs in the device order, on the engine's own export
        host_comp, Y_comp, Y_mean = X_comp, tr.device_attributes()["components"], mean_dev.reshape(1, -1)

    assert X_comp.shape[1] == sample_dims and X_comp.shape[0] == config.components \
        and X_global_mean.shape[1] == sample_dims and X_stdev.shape[0] == config.components, "Invalid shape"

    def random_projections():
        """random projections of the last group's buffer, centred on the global mean (:289-291,312-316)"""
        X_last = first if pooled else X
        n_rand_samples = min(5000, NB if large_d else X_last.shape[0])
        if device_dirs:
            # get_random_dirs' stream (RandomState(2).normal) drawn by the device generator: 42M normals at convs.4
            g = _native.legacy_normal([SEED_RANDOM_DIRS], config.components * sample_dims, device).view(config.components, -1)
            g = g / torch.linalg.vector_norm(g.double(), dim=1, keepdim=True).float()
            dirs_dev = g.view(config.components, lc, lh, lw).permute(0, 2, 3, 1).reshape(config.components, -1).contiguous()
        else:
            dirs_dev = pre_dirs
        if affine is not None:                                  # dirs . (x - mean) == (dirs Q) . (y - ybar)
            dirs_dev = _native.linear(dirs_dev, affine.Q.T.float().contiguous())
        sub = mean_dev
        if large_d:                                             # the engine centred the last group in place by its batch mean
            sub = mean_dev - tr.last_batch_mean()
            X_last = tr.last_batch_rows(n_rand_samples)         # (feature shards gathered when distributed)
        return _native.project_std(X_last[:n_rand_samples], dirs_dev, sub=sub)      # read back below, with lat_stdev

    # conv feature maps: the projections of the last batch come first, so that the regression's activations can then be written
    # over the engine's batch rows instead of into a [B, d] buffer of their own (33.5 GB at convs.8 and B = 2000).  Neither step
    # draws from a random state the other one reads, so the order changes no result.
    act_buf = None
    if large_d:
        rand_std_dev = random_projections()
        if layout is not None and not live and B <= tr._chain.nb_max:
            act_buf = tr._chain.batch_rows(B)
    if samples_are_latents:
        Z_comp = X_comp
        Z_global_mean = X_global_mean
    else:
        Z_comp, Z_global_mean = regression(Y_comp, Y_mean, X_stdev, inst, config, affine=affine, native=layout is not None,
                                           act_buf=act_buf, host_comp=host_comp)

    tick("export + regression")
    Z_comp /= np.linalg.norm(Z_comp, axis=-1, keepdims=True)
    if not large_d:
        rand_std_dev = random_projections()

    arrays = _final_arrays(config, X_comp, X_global_mean, X_stdev, X_var_ratio, Z_comp, Z_global_mean, rand_std_dev,
                           lambda: pre_lat if pre_lat is not None else model.sample_latent(5000).reshape(5000, input_dims),
                           sample_shape, input_shape, input_dims, (lambda A: A) if device_layout else to_nchw)
    if hasattr(model, "check_numerics"):
        model.check_numerics()
    tick("random directions + layout")
    if instrumented_model is None:
        inst.close()
        del inst
        del model
    return arrays


def get_or_compute(config, model=None, submit_config=None, force_recompute=False):
    if submit_config is None:
        wrkdir = str(Path(__file__).parent.resolve())
        submit_config = SimpleNamespace(run_dir_root=wrkdir, run_dir=wrkdir)
    return _compute(submit_config, config, model, force_recompute)


def _compute(submit_config, config, model=None, force_recompute=False):
    basedir = Path(submit_config.run_dir)

    if config.n is None:
        raise RuntimeError("Must specify number of samples with -n=XXX")
    if model and not isinstance(model, InstrumentedModel):
        raise RuntimeError('Passed model has to be wrapped in "InstrumentedModel"')
    if config.use_w and "StyleGAN" not in config.model:
        raise RuntimeError(f"Cannot change latent space of non-StyleGAN model {config.model}")

    dump_path = _dump_path(basedir, config)

    if not dump_path.is_file() or force_recompute:
        print("Not cached")
        t_start = datetime.datetime.now()
        compute(config, dump_path, model)
        print("Total time:", datetime.datetime.now() - t_start)
    return dump_path


def _dump_path(basedir, config):
    """The cache file of a decomposition: ``<run_dir>/cache/components/<model>-<class>_<layer>_<estimator>_n<n>[_w][_seed].npz``,
    named from the requested number of components."""
    transformer = get_estimator(config.estimator, config.components, config.sparsity)
    dump_name = "{}-{}_{}_{}_n{}{}{}.npz".format(
        config.model.lower(),
        config.output_class.replace(" ", "_"),
        config.layer.lower(),
        transformer.get_param_str(),
        config.n,
        "_w" if config.use_w else "",
        f"_seed{config.seed}" if config.seed else "",
    )
    return Path(basedir) / "cache" / "components" / dump_name


# ---- several layers in one pass -------------------------------------------------------------------------------------------
# bytes of activation rows (all layers together) whose statistics one set of launches computes in a multi-layer pass; a round
# of groups that holds more is split, which leaves every group's statistics unchanged
MULTI_ROWS_BYTES = 2 << 30


def get_or_compute_layers(config, layers, model=None, submit_config=None, force_recompute=False):
    """``get_or_compute`` for several layers of one model at once: returns ``{layer: path}``, each path the file that
    ``get_or_compute`` with ``config.layer = layer`` returns, with the same arrays.  Layers already in the cache are skipped
    unless ``force_recompute``.

    The layers share one draw of the latents, one activation run per microbatch (a ``partial_forward`` to the deepest of them
    with every layer retained), one grouped statistics launch per round and one regression pass; each layer keeps its own
    merge chain.  Every per-layer random stream is the one ``get_or_compute`` would draw, so the files are the per-layer files.

    Takes the layers a per-layer run decomposes with the small-d engine (d <= 1024) or through an exact affine factorisation
    (BigGAN ``generator.gen_z`` and its BatchNorm row layers), with ``--est ipca`` and a fixed ``batch_size``, in a single
    process.  ``config`` is not modified."""
    layers = list(layers)
    if len(set(layers)) != len(layers):
        raise ValueError(f"get_or_compute_layers: repeated layer names in {layers}")
    if config.n is None:
        raise RuntimeError("Must specify number of samples with -n=XXX")
    if model and not isinstance(model, InstrumentedModel):
        raise RuntimeError('Passed model has to be wrapped in "InstrumentedModel"')
    if config.use_w and "StyleGAN" not in config.model:
        raise RuntimeError(f"Cannot change latent space of non-StyleGAN model {config.model}")
    if config.estimator != "ipca":
        raise NotImplementedError(f"get_or_compute_layers: --est {config.estimator} is not available for several layers at once "
                                  "(only ipca); use get_or_compute per layer")
    if config.batch_size is None:
        raise ValueError("get_or_compute_layers needs a batch_size: the per-layer memory probe could pick a different B per layer")
    latents = [l for l in layers if l in ("g_mapping", "style") and config.use_w]
    if latents:
        raise ValueError(f"get_or_compute_layers: {latents} are the W latents themselves; they have no activation pass to "
                         "share: use get_or_compute")
    if _dist()[2]:
        raise NotImplementedError("get_or_compute_layers runs in a single process; use get_or_compute in a distributed job")
    if submit_config is None:
        wrkdir = str(Path(__file__).parent.resolve())
        submit_config = SimpleNamespace(run_dir_root=wrkdir, run_dir=wrkdir)
    configs = {}
    for layer in layers:
        configs[layer] = copy.copy(config)
        configs[layer].layer = layer
    paths = {layer: _dump_path(submit_config.run_dir, configs[layer]) for layer in layers}
    todo = [layer for layer in layers if force_recompute or not paths[layer].is_file()]
    if todo:
        print("Not cached:", ", ".join(todo))
        t_start = datetime.datetime.now()
        _compute_layers(config, todo, {layer: configs[layer] for layer in todo}, paths, model)
        print("Total time:", datetime.datetime.now() - t_start)
    return paths


def _compute_layers(config, layers, configs, paths, instrumented_model):
    """Runs the joint pass and writes every layer's file once all of them are computed (an interrupted or failed pass writes
    nothing)."""
    timestamp = lambda: datetime.datetime.now().strftime("%d.%m %H:%M")
    print(f"[{timestamp()}] Computing {len(layers)} layers in one pass")
    try:
        arrays = _layers_arrays(config, layers, instrumented_model)
    except _native.ChainNotConverged as err:
        # the status word is library-global: which layer's chain found no gap is not known.  Every layer runs again on its own,
        # each with compute()'s own retry through the direct chain step.
        print(f"{err}\nRe-running each layer on its own", flush=True)
        for layer in layers:
            compute(copy.copy(configs[layer]), paths[layer], instrumented_model)
        return
    for layer in layers:
        _write_npz(paths[layer], arrays[layer])


def _layers_arrays(config, layers, instrumented_model):
    """The 8 arrays of every layer, as ``compute_arrays`` computes them one layer at a time."""
    global B
    tick = _phase_timer()
    torch.manual_seed(0)
    np.random.seed(0)

    device = _native.require_cuda("cuda")
    if instrumented_model is None:
        inst = get_instrumented_model(config.model, config.output_class, list(layers),
                                      torch.device("cuda", torch.cuda.current_device()))
        model = inst.model
    else:
        print("Reusing InstrumentedModel instance")
        inst = instrumented_model
        model = inst.model
        inst.remove_edits()
        model.set_output_class(config.output_class)
    device = model.device
    if config.use_w:
        print("Using W latent space")
        model.use_w()

    # ---- the layers: exact affine factorisation or activations read from the hooks ----------------------------------------
    spec = {}
    for layer in layers:
        affine = model.affine_layer(layer) if hasattr(model, "affine_layer") else None
        spec[layer] = SimpleNamespace(affine=affine)
    act_layers = [l for l in layers if spec[l].affine is None]

    # ---- shape pass: one latent (the draw the per-layer run makes), every layer retained ----------------------------------
    inst.retain_layers(layers)
    z1 = model.sample_latent(1)

    def run_to(target):
        for l in layers:
            inst.retained_layer(l, clear=True)
        model.partial_forward(z1, target)
        return {l: v for l, v in inst.retained_features().items() if l in spec and v is not None}

    # the activation pass of every microbatch is one partial_forward to a layer whose run fills every activation layer
    deepest = None
    for target in reversed(act_layers):
        got = run_to(target)
        if all(l in got for l in act_layers):
            deepest = target
            break
    if act_layers and deepest is None:
        raise NotImplementedError(f"get_or_compute_layers: no partial_forward of {model.__class__.__name__} reaches all of "
                                  f"{act_layers}; use get_or_compute")
    shapes = {l: tuple(got[l].shape) for l in act_layers}
    for l in layers:
        if l not in shapes:
            shapes[l] = tuple(run_to(l)[l].shape)
    input_shape = inst.model.get_latent_shape()
    input_dims = int(inst.model.get_latent_dims())
    B = config.batch_size
    small_d_max = DeviceIncrementalPCA.SMALL_D_MAX
    for l in layers:
        s = spec[l]
        s.shape = shapes[l]
        s.dims = int(np.prod(s.shape))
        s.c = min(config.components, s.dims)
        print(f"{l}: feature shape {s.shape}")
        if s.affine is None and s.dims > small_d_max:
            raise NotImplementedError(f"get_or_compute_layers: {l} is a conv feature map (d = {s.dims} > {small_d_max}, the "
                                      "large-d engine); use get_or_compute")
        if s.affine is not None and s.c > s.affine.rank:
            raise NotImplementedError(f"components={s.c} exceeds the rank {s.affine.rank} of layer {l}")
        s.d = s.affine.Q.shape[1] if s.affine is not None else s.dims
        s.plan = _plan.make_plan(config.n, B, s.c)
        s.transformer = get_estimator(config.estimator, s.c, config.sparsity, device=device)
    print("B={}, N={}, layers={}".format(B, spec[layers[0]].plan.N, len(layers)), flush=True)

    # ---- Phase A: the seeds; each layer's are a prefix of the longest list (one global stream) ----------------------------
    torch.manual_seed(config.seed or SEED_SAMPLING)
    np.random.seed(config.seed or SEED_SAMPLING)
    seeds = _draw_seeds(max(spec[l].plan.n_calls for l in layers))

    # ---- Phase B: statistics + one merge chain per layer; layers whose plans agree (the same NB) share the pass -----------
    by_plan = {}
    for l in layers:
        by_plan.setdefault(spec[l].plan, []).append(l)
    for pl, members in by_plan.items():
        _fit_layers(model, inst, pl, members, spec, seeds, deepest, input_shape, input_dims, device)
    tick("sampling + activations + IPCA chains")

    # ---- per layer: export, affine lift and sign rule ---------------------------------------------------------------------
    for l in layers:
        s = spec[l]
        s.X_comp, s.X_stdev, s.X_var_ratio, s.mean_dev, s.X_global_mean, s.Y_comp, s.Y_mean = \
            _export_components(s.transformer, s.affine, False, s.dims, device)
        assert s.X_comp.shape[1] == s.dims and s.X_comp.shape[0] == s.c and s.X_global_mean.shape[1] == s.dims \
            and s.X_stdev.shape[0] == s.c, "Invalid shape"

    # ---- one regression pass for every layer ------------------------------------------------------------------------------
    Z = _linreg_layers(model, inst, config, layers, spec, deepest)
    tick("export + regression")

    # ---- per layer: random directions, lat_stdev, the arrays ---------------------------------------------------------------
    shared = {}

    def lat_samples():
        # the per-layer run draws these 5000 latents right after its regression pass: the same seed for every layer
        if "lat" not in shared:
            shared["lat"] = model.sample_latent(5000).reshape(5000, input_dims)
        return shared["lat"]

    out = {}
    for l in layers:
        s = spec[l]
        Z_comp, Z_global_mean = Z[l]
        Z_comp /= np.linalg.norm(Z_comp, axis=-1, keepdims=True)
        dirs = torch.from_numpy(get_random_dirs(s.c, s.dims)).to(device, non_blocking=True)
        if s.affine is not None:                            # dirs . (x - mean) == (dirs Q) . (y - ybar)
            dirs = _native.linear(dirs, s.affine.Q.T.float().contiguous())
        X = s.last_rows
        rand_std_dev = _native.project_std(X[:min(5000, X.shape[0])], dirs, sub=s.mean_dev)
        out[l] = _final_arrays(config, s.X_comp, s.X_global_mean, s.X_stdev, s.X_var_ratio, Z_comp, Z_global_mean, rand_std_dev,
                               lat_samples, s.shape, input_shape, input_dims, lambda A: A)
    if hasattr(model, "check_numerics"):
        model.check_numerics()
    tick("random directions")
    if instrumented_model is None:
        inst.close()
    return out


def _fit_layers(model, inst, pl, layers, spec, seeds, deepest, input_shape, input_dims, device):
    """Phase B of ``compute_arrays`` for several layers with one plan: the same chunks, rounds and groups; each microbatch's
    activations come from one partial_forward, each round's statistics from one grouped launch (tensor-core widths) plus
    batch_stats_multi (other widths), and each layer's chain steps through the groups in order on its own stream."""
    K, NB = pl.K, pl.NB
    groups_per_chunk = max(1, int(LATENT_CHUNK_BYTES // max(1, NB * input_dims * 4)))
    acts = [l for l in layers if spec[l].affine is None]
    grouped = [l for l in layers if _native.stats_grouped_width(spec[l].d)]
    per_group_bytes = NB * 4 * sum(spec[l].d for l in layers)
    span_max = max(1, MULTI_ROWS_BYTES // per_group_bytes)
    stopped = set()

    def layer_rows(rows):
        """{layer: [n, d] rows} for latent rows ``rows`` (n a multiple of NB), with compute_arrays' microbatches."""
        out = {l: spec[l].affine.coords(rows) for l in layers if spec[l].affine is not None}
        if acts:
            bufs = {l: torch.empty((rows.shape[0], spec[l].d), dtype=torch.float32, device=device) for l in acts}
            for g0 in range(0, rows.shape[0], NB):
                for mb in range(0, NB, B):
                    z = rows[g0 + mb:g0 + mb + B].reshape(-1, *input_shape[1:])
                    with torch.no_grad():
                        model.partial_forward(z, deepest)
                    feats = inst.retained_features()
                    space_left = min(B, NB - mb)
                    for l in acts:
                        bufs[l][g0 + mb:g0 + mb + space_left] = feats[l].reshape((z.shape[0], -1))[:space_left]
            out.update(bufs)
        return out

    for c0 in range(0, K, groups_per_chunk):
        c1 = min(c0 + groups_per_chunk, K)
        runs = _plan.contiguous_runs(_plan.groups_to_process(pl, 0, 1, c0, c1))
        needed, offsets = _plan.batch_slots(pl, runs)
        lat, ensure_rows = _sample_batches_lazy(model, B, [seeds[b] for b in needed])
        lat = lat.reshape(lat.shape[0], -1)
        where = {kk: off + (kk - run[0]) * NB for run, off in zip(runs, offsets) for kk in run}
        for rnd in _plan.rounds(c0, c1, 1, STATS_FIRST_BLOCK if c0 == 0 else STATS_BLOCK, STATS_BLOCK):
            for s0 in range(0, len(rnd), span_max):
                span = list(rnd)[s0:s0 + span_max]
                r0 = where[span[0]]
                assert all(where[kk] == r0 + i * NB for i, kk in enumerate(span))
                ensure_rows(r0 + len(span) * NB)
                X = layer_rows(lat[r0:r0 + len(span) * NB])
                stats = dict(zip(grouped, _native.batch_stats_grouped([(X[l], len(span), NB, None, None) for l in grouped])))
                for l in layers:
                    if l not in stats:
                        stats[l] = _native.batch_stats_multi(X[l], len(span), NB)
                    spec[l].last_rows = X[l][(len(span) - 1) * NB:]
                for i in range(len(span)):
                    for l in layers:
                        if l not in stopped and not spec[l].transformer.fit_partial_stats(NB, stats[l][0][i], stats[l][1][i]):
                            stopped.add(l)      # the per-layer loop leaves its fit here (n_components > first batch)
        ensure_rows(lat.shape[0])
        del lat


def _linreg_layers(model, inst, config, layers, spec, deepest):
    """``linreg_lstsq`` for every layer from one pass over the SEED_LINREG latents: {layer: (Z_comp, Z_mean)}."""
    for l in layers:
        _warn_if_not_orthonormal(spec[l].Y_comp)
    print("Performing least squares regression", flush=True)
    torch.manual_seed(SEED_LINREG)
    np.random.seed(SEED_LINREG)
    dev = model.device
    ops = {}
    for l in layers:
        s = spec[l]
        ops[l] = (torch.from_numpy(s.Y_comp).float().to(dev).contiguous(),
                  torch.from_numpy(s.Y_mean).float().to(dev).reshape(-1).contiguous(),
                  torch.from_numpy(s.X_stdev).float().to(dev).contiguous())
    n_samp = max(10_000, config.n) // B * B
    latent_dims = int(model.get_latent_dims())      # consumes one global draw, as in the reference (:88)
    accs = {l: _native.LinregAccumulator(ops[l][0].shape[0], latent_dims, dev) for l in layers}
    acts = [l for l in layers if spec[l].affine is None]
    seeds = _draw_seeds(n_samp // B)
    group = max(1, min(len(seeds), (256 << 20) // max(1, B * latent_dims * 4)))
    for start in range(0, len(seeds), group):
        idx = list(range(start, min(start + group, len(seeds))))
        z_all = _sample_batches(model, B, [seeds[i] for i in idx])
        for j in range(len(idx)):
            z = z_all[j * B:(j + 1) * B]
            if acts:
                with torch.no_grad():
                    model.partial_forward(z, deepest)
                feats = inst.retained_features()
            for l in layers:
                if spec[l].affine is not None:
                    act = spec[l].affine.coords(z.reshape(B, -1))
                else:
                    act = feats[l].reshape(B, -1)
                accs[l].accumulate(act.contiguous(), *ops[l], z.reshape(B, -1).contiguous())
    out = {}
    for l in layers:
        accs[l].n_total = n_samp
        M_t, Z_mean = accs[l].solve()
        out[l] = (M_t.cpu().numpy()[:ops[l][0].shape[0], :], Z_mean.cpu().numpy().reshape(1, -1))
    return out
