"""Estimators of the hot path: ``IPCAEstimator`` / ``get_estimator``.

Mirror of /root/reference/estimators.py:55-81,206-218.  ``IPCAEstimator`` keeps the reference's
interface (``batch_support``, ``get_param_str``, ``fit``, ``fit_partial``, ``get_components`` and a
``.transformer`` object exposing scikit-learn's fitted attributes ``mean_``, ``var_``, ``components_``,
``singular_values_``, ``explained_variance_``, ``explained_variance_ratio_``, ``n_samples_seen_``) but the
arithmetic of ``IncrementalPCA.partial_fit`` runs on the device: per-batch statistics (csrc/stats.cu)
feed the fp64 Gram-form merge chain (csrc/ipca.cu).  Batches may be host ndarrays (copied in, as the
reference API allows) or CUDA tensors (no copy: the samples never leave HBM).  For d > 1024 (conv feature
maps) the d x d Gram is out of reach and the small-side engine (csrc/bigd.cu) takes over behind the same
interface; its stacked matrix lives in HBM and producers can write batches in place (``batch_buffer``).

``FacebookPCAEstimator`` (estimators.py:120-160, fbpca.pca with raw=True) runs on the device from pooled batch statistics
(csrc/rsvd.cu): its fit depends on the stacked samples only through their d x d Gram, so the driver never materialises them.
The remaining estimators of the reference (pca / ica / spca, estimators.py:18-52,84-118,162-204) are not batched and appear
in no BASELINE config; asking for them raises (SURVEY.md section 2 marks them out of scope).
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import torch

from . import _native


class DeviceIncrementalPCA:
    """The ``.transformer`` of IPCAEstimator: sklearn's fitted-attribute names, device-resident state."""

    def __init__(self, n_components, whiten=False, batch_size=None, device=None):
        if whiten:
            raise NotImplementedError("whiten=True is not used by GANSpace (estimators.py:58)")
        self.n_components = n_components
        self.whiten = whiten
        self.batch_size = batch_size
        self._device = device
        self._chain = None
        self._host = None            # cached export (host view)
        self._dev = None             # ... and its device tensors
        self._shard = None           # (rank, world): feature-sharded large-d engine (SURVEY.md section 8e)
        self._stage = None
        self.host_layout = None      # large-d engine: (hw, c) of NHWC rows -- components_ / mean_ are read back in NCHW order
        self.n_samples_seen_ = np.int64(0)

    def enable_feature_sharding(self, rank, world):
        """Large-d engine over a torch.distributed job: every rank keeps d/world features of the stacked matrix and
        produces nb/world rows of each batch; ``partial_fit_inplace`` exchanges them with one all-to-all."""
        if self._chain is not None:
            raise RuntimeError("enable_feature_sharding must precede the first partial_fit")
        self._shard = (int(rank), int(world)) if world > 1 else None

    # -- device side ---------------------------------------------------------------------------------
    SMALL_D_MAX = 1024          # above this the d x d Gram engine (csrc/ipca.cu) gives way to the small-side engine (bigd.cu)

    def _ensure(self, d, device, nb=None):
        if self._chain is None:
            if self.n_components > d:
                raise ValueError(
                    "n_components=%r invalid for n_features=%d, need more rows than columns for "
                    "IncrementalPCA processing" % (self.n_components, d))
            if d > self.SMALL_D_MAX:
                self._chain = _native.BigIPCA(d, self.n_components, nb, device, shard=self._shard)
            else:
                self._chain = _native.IPCAChain(d, self.n_components, device)
        elif getattr(self._chain, "d_full", self._chain.d) != d:     # (a feature-sharded engine's .d is its local width)
            raise ValueError("Number of input features has changed from %i to %i between calls to partial_fit!"
                             % (getattr(self._chain, "d_full", self._chain.d), d))
        return self._chain

    @property
    def is_large_d(self):
        return isinstance(self._chain, _native.BigIPCA)

    def batch_buffer(self, nb, d, device):
        """Large-d engine only: the [nb, d] rows of the device-resident stacked matrix that the NEXT partial_fit will
        consume.  Producers (e.g. the synthesis kernels) write the raw batch there; then ``partial_fit_inplace(nb)``."""
        if d <= self.SMALL_D_MAX:
            raise ValueError("batch_buffer is the large-d engine's interface (d > %d)" % self.SMALL_D_MAX)
        chain = self._ensure(int(d), device, nb=int(nb))
        if self._shard is not None:
            # sharded: the caller fills a staging buffer with ITS rows [rank*q, (rank+1)*q) of the batch, all d features
            world = self._shard[1]
            if nb % world != 0 or nb > chain.nb_max:
                raise ValueError(f"feature-sharded IPCA needs equal batches divisible by the world size (nb={nb}, world={world})")
            q = nb // world
            if self._stage is None or self._stage.shape != (q, int(d)):
                self._stage = torch.empty((q, int(d)), dtype=torch.float32, device=chain.dev)
            return self._stage
        if nb > chain.nb_max:                                   # a later batch larger than the first: grow, keep the state
            big = _native.BigIPCA(chain.d, chain.c, int(nb), chain.dev, gram="tc" if chain.flags & 1 else "simt")
            big.M[:chain.c].copy_(chain.M[:chain.c])
            big.state.copy_(chain.state)
            big.n_seen = chain.n_seen
            self._chain = chain = big
        return chain.batch_rows(int(nb))

    def partial_fit_inplace(self, nb):
        chain = self._chain
        if int(self.n_samples_seen_) == 0 and self.n_components > nb:
            raise ValueError(f"n_components={self.n_components} must be less or equal to the batch number of "
                             f"samples {nb} for the first partial_fit call.")
        if self._shard is not None:
            _native.exchange_rows(self._stage, chain.batch_rows(int(nb)), self._shard[1])
        chain.step(int(nb))          # centres the batch rows in place (chain.batch_mean holds the batch mean)
        self.n_samples_seen_ = np.int64(chain.n_seen)
        self._host = None
        return self

    def batch_stats(self, X):
        """(n, mean[d], centred Gram[d,d]) of a batch; host arrays are copied to the device first."""
        if isinstance(X, np.ndarray):
            dev = _native.require_cuda(self._device)
            X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
        if X.dim() != 2:
            raise ValueError("Expected 2D array, got %dD" % X.dim())
        if X.dtype != torch.float32:
            X = X.float()
        mean, gram = _native.batch_stats(X)
        return int(X.shape[0]), mean, gram

    def merge(self, n_batch, mean_b, gram_b):
        """One partial_fit step from precomputed batch statistics (must follow the reference's batch order)."""
        chain = self._ensure(int(mean_b.shape[0]), mean_b.device)
        if int(self.n_samples_seen_) == 0 and self.n_components > n_batch:
            raise ValueError(f"n_components={self.n_components} must be less or equal to the batch number of "
                             f"samples {n_batch} for the first partial_fit call.")
        chain.step(n_batch, mean_b, gram_b)
        self.n_samples_seen_ = np.int64(chain.n_seen)
        self._host = None

    def partial_fit(self, X, y=None):
        d = int(X.shape[1]) if getattr(X, "ndim", 2) == 2 else 0
        if d > self.SMALL_D_MAX:
            if isinstance(X, np.ndarray):
                X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32))
            dev = X.device if X.is_cuda else _native.require_cuda(self._device)
            self.batch_buffer(X.shape[0], d, dev).copy_(X)      # host arrays are copied in, CUDA tensors stay in HBM
            return self.partial_fit_inplace(X.shape[0])
        self.merge(*self.batch_stats(X))
        return self

    # -- saved state (decomposition.get_or_extend) ------------------------------------------------------
    def state_dict(self):
        """The engine after the batches merged so far, as host arrays (one device -> host copy per blob) plus its sizes:
        ``engine`` is 'ipca' (small-d chain) or 'bigd' (large-d engine, with its batch size ``nb``)."""
        if self._chain is None:
            raise AttributeError("IncrementalPCA is not fitted yet")
        if self._shard is not None:
            raise NotImplementedError("a feature-sharded engine's state is not saved")
        sd = self._chain.state_dict()
        sd.update(engine="bigd" if self.is_large_d else "ipca", d=int(self._chain.d), c=int(self.n_components))
        if self.is_large_d:
            sd["nb"] = int(self._chain.nb_max)
        return sd

    def load_state_dict(self, sd, device=None):
        """Continue from ``state_dict()``: the engine is created for its (d, nb) if there is none yet."""
        if int(sd["c"]) != self.n_components:
            raise ValueError(f"saved state has {sd['c']} components, this estimator {self.n_components}")
        chain = self._ensure(int(sd["d"]), device if device is not None else self._device, nb=sd.get("nb"))
        if (sd["engine"] == "bigd") != self.is_large_d:
            raise ValueError(f"saved state of the {sd['engine']} engine does not fit this one")
        chain.load_state_dict(sd)
        self.n_samples_seen_ = np.int64(chain.n_seen)
        self._host = None
        return self

    def centre_last_batch(self):
        """Large-d engine after ``load_state_dict``: its producer has written the last batch's raw rows again into
        ``batch_buffer``; centre them by the saved batch mean exactly as the step did (float32 of the fp64 difference), so that
        ``last_batch_rows`` is what it was after that step, without stepping."""
        ch = self._chain
        rows = ch.batch_rows(ch.last_nb)
        step = max(1, (256 << 20) // (8 * rows.shape[1]))
        for r0 in range(0, rows.shape[0], step):
            blk = rows[r0:r0 + step]
            blk.copy_((blk.double() - ch.batch_mean[None, :]).float())

    def last_batch_mean(self):
        """Large-d engine: fp64 [d] mean of the batch the last partial_fit centred in place."""
        return self._chain.gathered(self._chain.batch_mean.unsqueeze(0)).reshape(-1)

    def last_batch_rows(self, n):
        """Large-d engine: the first n rows of the last batch as centred by partial_fit, full feature width."""
        return self._chain.gathered(self._chain.batch_rows(self._chain.last_nb)[:n])

    # -- sklearn attribute names (host copies, fetched lazily) ---------------------------------------
    def device_attributes(self):
        """sklearn's fitted attributes as device tensors; one export per fit state (the host view below reuses it)."""
        if self._chain is None:
            raise AttributeError("IncrementalPCA is not fitted yet")
        if self._host is None or self._dev is None:
            self._dev = self._chain.export()
        return self._dev

    def _export(self):
        if self._chain is None:
            raise AttributeError("IncrementalPCA is not fitted yet")
        if self._host is None:
            dev = self._chain.export()
            # ONE device->host transfer: the six arrays packed into one fp64 buffer (each .cpu() is a synchronising copy)
            keys = list(dev)
            if sum(dev[k].numel() for k in keys) <= (1 << 22):
                flat = torch.cat([dev[k].reshape(-1).double() for k in keys]).cpu().numpy()
                host, off = {}, 0
                for k in keys:
                    n = dev[k].numel()
                    host[k] = flat[off:off + n].reshape(tuple(dev[k].shape)).astype(
                        np.float32 if dev[k].dtype == torch.float32 else np.float64)
                    off += n
            elif self.host_layout is not None:
                # conv feature maps in the producers' NHWC order: components and mean are permuted to the reference's NCHW
                # order on the device (gsb_nhwc_to_nchw_rows), then copied once; the device tensors keep the NHWC order
                hw, ch = self.host_layout
                host = {}
                for k, v in dev.items():
                    if k in ("components", "mean", "var"):
                        host[k] = _native.nhwc_to_nchw_rows(v.reshape(-1, hw * ch), hw, ch).cpu().numpy().reshape(v.shape)
                    else:
                        host[k] = v.cpu().numpy()
            else:                                        # conv feature maps: 168 MB of components, copied as they are
                host = {k: v.cpu().numpy() for k, v in dev.items()}
            self._dev = dev
            self._host = host
        return self._host

    components_ = property(lambda self: self._export()["components"])
    singular_values_ = property(lambda self: self._export()["singular_values"])
    mean_ = property(lambda self: self._export()["mean"])
    var_ = property(lambda self: self._export()["var"])
    explained_variance_ = property(lambda self: self._export()["explained_variance"])
    explained_variance_ratio_ = property(lambda self: self._export()["explained_variance_ratio"])


class IPCAEstimator:
    def __init__(self, n_components, device=None):
        self.n_components = n_components
        self.whiten = False
        self.transformer = DeviceIncrementalPCA(n_components, whiten=self.whiten,
                                                batch_size=max(100, 2 * n_components), device=device)
        self.batch_support = True

    def get_param_str(self):
        return "ipca_c{}{}".format(self.n_components, "_w" if self.whiten else "")

    def fit(self, X):
        # sklearn IncrementalPCA.fit: partial_fit over gen_batches(n, batch_size, min_batch_size=n_components)
        n = X.shape[0]
        bs = self.transformer.batch_size
        start = 0
        while start < n:
            end = start + bs
            if end + self.n_components > n:
                end = n
            self.transformer.partial_fit(X[start:end])
            start = end

    def fit_partial(self, X):
        try:
            self.transformer.partial_fit(X)
            self.transformer.n_samples_seen_ = np.int64(self.transformer.n_samples_seen_)   # estimators.py:71-72
            return True
        except ValueError as e:
            print("\nIPCA error:", e)
            return False

    def fit_partial_stats(self, n_batch, mean_b, gram_b):
        """fit_partial from the batch's sufficient statistics (n, mean [d], centred Gram [d, d]; fp64 device tensors)
        instead of its rows -- small-d engine; must be called in the reference's batch order."""
        try:
            self.transformer.merge(int(n_batch), mean_b, gram_b)
            self.transformer.n_samples_seen_ = np.int64(self.transformer.n_samples_seen_)
            return True
        except ValueError as e:
            print("\nIPCA error:", e)
            return False

    def fit_partial_inplace(self, nb):
        """fit_partial on the batch already written into ``transformer.batch_buffer(nb, d, device)`` (large-d engine)."""
        try:
            self.transformer.partial_fit_inplace(nb)
            return True
        except ValueError as e:
            print("\nIPCA error:", e)
            return False

    def state_dict(self):
        return self.transformer.state_dict()

    def load_state_dict(self, sd, device=None):
        self.transformer.load_state_dict(sd, device)

    def get_components(self):
        stdev = np.sqrt(self.transformer.explained_variance_)
        var_ratio = self.transformer.explained_variance_ratio_
        return self.transformer.components_, stdev, var_ratio


class FacebookPCAEstimator:
    """fbpca.pca(X, k=c, n_iter=2, raw=True, l=2c) on the device (reference estimators.py:124-160).

    ``fit(X)`` takes the whole sample matrix (host ndarray or CUDA tensor, d <= 1024).  The driver instead feeds per-group
    statistics (``fit_partial_stats``, in the reference's row order), pads with the zero rows of its unfilled sample matrix
    (``add_zero_rows``) and calls ``fit_pooled``; the samples are never stacked.  fbpca's test matrix Omega is drawn from
    NumPy's global state (``draw_omega``), exactly as fbpca draws it, unless the caller passes one."""

    SMALL_D_MAX = DeviceIncrementalPCA.SMALL_D_MAX

    def __init__(self, n_components, device=None):
        self.n_components = n_components
        self.transformer = SimpleNamespace()
        self.batch_support = False
        self.n_iter = 2
        self.l = 2 * self.n_components
        self._device = device
        self._pool = None
        self.stdev = None
        self.total_var = None
        self.var_ratio = None
        self.device_outputs = None

    def get_param_str(self):
        return "fbpca_c{}_it{}_l{}".format(self.n_components, self.n_iter, self.l)

    def randomized(self, m, d):
        """fbpca's branch choice for an [m, d] matrix: False = exact SVD (l >= m/1.25 or l >= d/1.25)."""
        return not (self.l >= m / 1.25 or self.l >= d / 1.25)

    def draw_omega(self, m, d):
        """fbpca's test matrix for an [m, d] matrix (m >= d): np.random.uniform(-1, 1, (d, l)) cast to float32, drawn from the
        global NumPy state -- or None for the exact branch, which draws nothing."""
        if not self.randomized(m, d):
            return None
        return np.random.uniform(low=-1.0, high=1.0, size=(d, self.l)).astype(np.float32)

    def _ensure(self, d, device):
        if self._pool is None:
            if not (32 <= d <= self.SMALL_D_MAX and d % 32 == 0):
                raise NotImplementedError(f"fbpca runs on the device for 32 <= d <= {self.SMALL_D_MAX}, d % 32 == 0 (d={d})")
            self._pool = _native.FBPCAPool(d, _native.require_cuda(device if device is not None else self._device))
        elif self._pool.d != d:
            raise ValueError(f"Number of input features has changed from {self._pool.d} to {d}")
        return self._pool

    def fit_partial_stats(self, n_batch, mean_b, gram_b):
        """Pool one group's statistics (n, mean [d], centred Gram [d, d]; fp64 device tensors), in the reference's row order."""
        pool = self._ensure(int(mean_b.shape[-1]), mean_b.device)
        pool.accumulate(int(n_batch), mean_b.reshape(1, -1).contiguous(), gram_b.contiguous())
        return True

    def add_zero_rows(self, n_zero):
        self._pool.add_zero_rows(int(n_zero))

    def state_dict(self):
        """The pool of the groups folded so far (save it before ``add_zero_rows``: the zero rows depend on the final N)."""
        if self._pool is None:
            raise AttributeError("nothing pooled yet")
        sd = self._pool.state_dict()
        sd.update(engine="fbpca", d=int(self._pool.d), c=int(self.n_components))
        return sd

    def load_state_dict(self, sd, device=None):
        if int(sd["c"]) != self.n_components:
            raise ValueError(f"saved state has {sd['c']} components, this estimator {self.n_components}")
        self._pool = None
        self._ensure(int(sd["d"]), device).load_state_dict(sd)

    def fit_pooled(self, omega=None, raw=False):
        """fbpca.pca on the pooled samples: ``raw`` = False when they were centred (the driver: X = samples - mean, so
        X^T X is the centred scatter), True for fbpca's raw=True on uncentred rows.  ``omega`` [d, l] (None = exact branch)."""
        pool = self._pool
        c, d = self.n_components, pool.d
        if not (1 <= c <= min(pool.n, d)):
            raise ValueError(f"n_components={c} must be in [1, min(n_samples, n_features)] = [1, {min(pool.n, d)}]")
        if omega is not None:
            omega = torch.as_tensor(np.asarray(omega, dtype=np.float64) if isinstance(omega, np.ndarray) else omega)
        self._finish(pool.solve(c, self.l, omega=omega, raw=raw), raw)

    def fit_pooled_affine(self, omega, Q, rank):
        """fit_pooled for samples pooled in the coordinates of a basis: activation rows x = y Q^T with Q [D, d] (fp64 device,
        orthonormal columns, zero padding columns allowed) and y the pooled d-vectors, the stacked matrix of rank ``rank``.
        ``omega`` [D, l]: fbpca's test matrix of the D-wide activations (None: its exact branch).  fbpca depends on Omega only
        through range(G^2 Omega) = Q range(G_y^2 Q^T Omega) (G = Q G_y Q^T): for l < rank the randomized solve runs on the pool
        with Q^T Omega; for l >= rank that range is all of range(G), so fbpca's result is the exact top-c PCA (DESIGN.md
        section 5g).  Components, mean and the sign rule stay in y-coordinates (the caller lifts them); stdev and var_ratio
        are those of the activations, Q being an isometry on the pooled rows."""
        c, pool = self.n_components, self._pool
        if not (1 <= c <= min(pool.n, rank)):
            raise ValueError(f"n_components={c} must be in [1, min(n_samples, rank)] = [1, {min(pool.n, rank)}]")
        omega_y = None
        if omega is not None and self.l < rank:
            omega_y = _native.fbpca_project_omega(Q, torch.as_tensor(omega).to(Q.device, torch.float32))
        self._finish(pool.solve(c, self.l, omega=omega_y), raw=False)

    def _finish(self, out, raw):
        c, d = self.n_components, self._pool.d
        self.device_outputs = out
        flat = torch.cat([out["components"].reshape(-1), out["stdev"], out["var_ratio"], out["mean"]]).cpu().numpy()
        comp, rest = flat[:c * d].reshape(c, d), flat[c * d:]
        self.transformer.components_ = comp
        self.stdev = rest[:c]
        self.var_ratio = rest[c:2 * c]
        self.total_var = float(self.stdev[0] ** 2 / self.var_ratio[0]) if self.var_ratio[0] > 0 else 0.0
        mean = rest[2 * c:].reshape(1, d)
        # X.mean(0) of the matrix fbpca saw: the raw rows' mean, or ~0 when the driver centred them
        self.transformer.mean_ = mean if raw else np.zeros_like(mean)
        self.pooled_mean = mean
        dotps = comp @ comp.T - np.eye(c)
        if not np.allclose(dotps, 0, atol=1e-4):
            print("FBPCA components not orghogonal, max dot", np.abs(dotps).max())

    def fit(self, X, omega=None):
        """fbpca.pca(X, k=c, n_iter=2, raw=True, l=2c) for an [m, d] matrix with m >= d (host ndarray or CUDA tensor)."""
        if isinstance(X, np.ndarray):
            X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(_native.require_cuda(self._device))
        if X.dim() != 2:
            raise ValueError("Expected 2D array, got %dD" % X.dim())
        m, d = int(X.shape[0]), int(X.shape[1])
        if m < d:
            raise NotImplementedError("fbpca on the device covers m >= n (more samples than features)")
        self._pool = None
        pool = self._ensure(d, X.device)
        mean, gram = _native.batch_stats(X.float().contiguous())
        pool.accumulate(m, mean.reshape(1, d), gram.reshape(1, d, d))
        if omega is None:
            omega = self.draw_omega(m, d)
        elif not self.randomized(m, d):
            omega = None
        self.fit_pooled(omega=omega, raw=True)

    def get_components(self):
        return self.transformer.components_, self.stdev, self.var_ratio


def get_estimator(name, n_components, alpha, device=None):
    if name == "ipca":
        return IPCAEstimator(n_components, device=device)
    if name == "fbpca":
        return FacebookPCAEstimator(n_components, device=device)
    if name in ("pca", "ica", "spca"):
        raise RuntimeError(f"estimator '{name}' is not batched and outside the GPU hot path "
                           "(SURVEY.md section 2); use 'ipca'")
    raise RuntimeError("Unknown estimator")
