"""GPU probe of the fp64 eigensolver (`gsb_sym_eig_top`): accuracy vs LAPACK and event-timed cost per call, for every
tridiagonalisation branch.

Each (d, c) case runs on two seeded matrices: a decaying spectrum, and a zero-padded rank-deficient one shaped like the
large-d engine's first-step T (only rows/columns c .. c+m-1 live, rank m-1), which reaches the sigma == 0 / beta == 0 paths.

    python tools/eig_probe.py [--lib path/to/libganspace_b200.so] [--out eig.npz] [--reps 20]

`--out` dumps every case's eigenvalues and eigenvectors, so that two builds can be compared bit for bit.
"""
import argparse
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from ganspace_b200 import _native as nat  # noqa: E402

CASES = [(96, 12), (128, 8), (256, 16), (352, 24), (512, 80), (640, 80), (672, 80), (992, 80), (1024, 40), (2112, 80),
         (4096, 128)]


def decaying(d, c):
    rng = np.random.RandomState(d + c)
    B = rng.standard_normal((d, 3 * d)) * (0.97 ** np.arange(d))[:, None]
    return B @ B.T


def padded(d, c):
    rng = np.random.RandomState(7 * d + c)
    m = (d - c) // 2
    X = rng.standard_normal((m, 2 * m)) * (0.99 ** np.arange(2 * m))[None, :]
    X -= X.mean(axis=0)
    A = np.zeros((d, d))
    A[c:c + m, c:c + m] = X @ X.T
    return A


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="libganspace_b200.so to load instead of the in-tree build")
    ap.add_argument("--out", help="write every case's (evals, evecs) to this .npz")
    ap.add_argument("--reps", type=int, default=20, help="timed calls per case")
    args = ap.parse_args()
    if args.lib:
        nat._LIB_PATH = Path(args.lib).resolve()
    lib = nat.load()
    dev = torch.device("cuda:0")
    dump = {}
    for d, c in CASES:
        for kind, make in (("decay", decaying), ("padded", padded)):
            A = make(d, c)
            lam, Q = np.linalg.eigh(A)
            lam, Q = lam[::-1][:c], Q[:, ::-1][:, :c].T
            At = torch.tensor(A, device=dev)
            ev, evec = nat.sym_eig_top(At, c)
            ev, evec = ev.cpu().numpy(), evec.cpu().numpy()
            dump[f"d{d}_c{c}_{kind}_evals"], dump[f"d{d}_c{c}_{kind}_evecs"] = ev, evec
            scale = max(lam[0], 1e-300)
            R = A @ evec.T - evec.T * ev[None, :]
            line = (f"d={d} c={c} {kind}: eval err {np.max(np.abs(ev - lam)) / scale:.2e} "
                    f"resid {np.max(np.linalg.norm(R, axis=0)) / scale:.2e} orth {np.max(np.abs(evec @ evec.T - np.eye(c))):.2e}")
            if kind == "decay":
                line += f" min|cos| {np.min(np.abs(np.sum(evec * Q, axis=1))):.10f}"
            ws = torch.empty(lib.gsb_ipca_workspace_bytes(d, c), dtype=torch.uint8, device=dev)
            evals = torch.empty(c, dtype=torch.float64, device=dev)
            evecs = torch.empty((c, d), dtype=torch.float64, device=dev)
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

            def call():
                rc = lib.gsb_sym_eig_top(C.c_void_p(At.data_ptr()), d, c, C.c_void_p(evals.data_ptr()),
                                         C.c_void_p(evecs.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), st)
                assert rc == 0, lib.gsb_last_error().decode()
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                call()
            e1.record()
            torch.cuda.synchronize()
            print(f"{line}  {e0.elapsed_time(e1) / args.reps * 1e3:.1f} us per call", flush=True)
            nat.check_eig_status("probe")
    if args.out:
        np.savez(args.out, **dump)


if __name__ == "__main__":
    main()
