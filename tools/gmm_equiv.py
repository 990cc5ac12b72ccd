"""Bit-identity of the full-covariance Gaussian mixture across two builds of the library.

    python tools/gmm_equiv.py dump FILE.npz       # on the build to compare against
    python tools/gmm_equiv.py compare FILE.npz    # on the build under test: every array np.array_equal

Records every output of gmm_fit(X, K, ...) with the default covariance_type ('full', AM_GMM_FULL) and
intermediates=True, except the phase times: the weights, means, covariances, precision factors, bounds, n_iter,
converged, best init, labels, k-means++ rows and every init's bounds, iterations and convergence.  The inputs are
tests/test_gpu_gmm.py's full-fit sets (ragged N, d up to 256, K in {1, 2, 40, 100}, N = K, overlap, duplicated rows)
with n_init = 10 and random_state = 21, and its task shape (20 000 x 200, K = 60, n_init = 1, 3 iterations, tol = 0).
gmm_fit is called without the covariance_type argument so that the same script runs on builds that predate it.
Needs an H100."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiomuse_ai_b200 import clustering_gpu as cg  # noqa: E402
from tests.test_gpu_gmm import FULL_SETS, SEED, blobs  # noqa: E402

FIELDS = ("weights", "means", "covariances", "precisions_cholesky", "lower_bounds", "n_iter", "converged", "best_init",
          "labels", "kpp", "init_lower_bounds", "init_n_iter", "init_converged")


def _record(key, f):
    return {f"{key}/{n}": np.asarray(getattr(f, n)) for n in FIELDS}


def _collect():
    out = {}
    for name, N, d, K, spread, dup in FULL_SETS:
        X = blobs(sum(map(ord, name)), N, d, K, spread=spread, dup=dup)
        out.update(_record(name, cg.gmm_fit(X, K, n_init=10, random_state=SEED, intermediates=True)))
    rng = np.random.default_rng(9)
    X = rng.standard_normal((20000, 200)) + np.repeat(rng.standard_normal((60, 200)), 334, 0)[:20000]
    X = (X - X.mean(0)) / X.std(0)
    out.update(_record("task_shape", cg.gmm_fit(X, 60, n_init=1, max_iter=3, tol=0.0, random_state=1,
                                                intermediates=True)))
    return out


def main():
    mode, path = sys.argv[1], sys.argv[2]
    got = _collect()
    if mode == "dump":
        np.savez(path, **got)
        print(f"wrote {len(got)} arrays to {path}")
        return 0
    want = np.load(path)
    bad = [k for k in sorted(set(want.files) | set(got))
           if not (k in got and k in want.files and np.array_equal(want[k], got[k], equal_nan=True))]
    for k in bad:
        print(f"DIFFERENT: {k}")
    print(f"{len(got) - len(bad)} of {len(got)} arrays equal, {len(bad)} different")
    return 1 if bad or len(got) != len(want.files) else 0


if __name__ == "__main__":
    sys.exit(main())
