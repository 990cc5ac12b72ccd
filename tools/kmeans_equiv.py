"""Equivalence of the k-means entry points across two builds of the library.

    python tools/kmeans_equiv.py dump FILE.npz       # on the build to compare against
    python tools/kmeans_equiv.py compare FILE.npz    # on the build under test

Seeded shapes on both sides of every boundary of the Lloyd-step choice (kmeans_use_tensor_cores in kmeans.cu):
k of 1, 7, 16, 128, 129 and 200; d of 1, 58, 200, 512, 4096 and 4097 (d % 4 != 0 included); N never a multiple of
128, and N k d just below and just above 5e7 (a fit) and 2e9 (a one-shot assignment).  Each shape goes through
am_kmeans_assign_dev, a plan step (sums, counts, inertia, dist) and an inertia-only plan step, am_kmeans_fit from
given centres and a seeded am_kmeans_fit with n_init = 2.  Per call: every output, and the kernels launched with
their counts (am_profile_report, template arguments stripped).

compare: kernel lists, the plan's path, and every single-step labels, counts and dist must be identical.  Sums,
inertia and fit outputs pass through float atomics, so they are judged by the tests' tolerances: sums rtol 2e-5
(atol 2e-3), inertia 1e-5 relative, fit labels > 0.999 equal, fit centres within 1e-4 of their scale, n_iter within
one step; a fit's clusters are matched to the other build's nearest centres first.  Compare a build with its own
second run first: that is the noise the tolerances must cover.  Needs an H100."""
import ctypes as C
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiomuse_ai_b200 import _lib, clustering_gpu as cg  # noqa: E402

# (N, d, k): N k d of the boundary pairs = 15 623 / 15 627 x 200 x 16 around 5e7, 30 517 / 30 518 x 512 x 128
# around 2e9
SHAPES = ((1001, 1, 1), (3001, 58, 7), (5003, 200, 16), (2001, 512, 128), (2001, 512, 129), (1501, 200, 200),
          (301, 4096, 16), (301, 4097, 16), (999, 4097, 7), (15623, 200, 16), (15627, 200, 16), (30517, 512, 128),
          (30518, 512, 128))
FIT_ITERS = 8


def _kernels():
    """Kernels launched since the last call: 'name:count', template arguments and parentheses stripped."""
    agg = {}
    for name, v in _lib.profile_report().items():
        while re.search(r"<[^<>]*>", name):
            name = re.sub(r"<[^<>]*>", "", name)
        name = name.strip("() ")
        agg[name] = agg.get(name, 0) + int(v["count"])
    return np.array(sorted(f"{k}:{c}" for k, c in agg.items()))


def _data(N, d, k, seed):
    rng = np.random.default_rng(seed)
    cen = rng.standard_normal((k, d)).astype(np.float32) * 3
    x = cen[rng.integers(0, k, N)] + rng.standard_normal((N, d)).astype(np.float32)
    init = x[rng.choice(N, k, replace=False)] + 0.1 * rng.standard_normal((k, d)).astype(np.float32)
    return np.ascontiguousarray(x, np.float32), np.ascontiguousarray(init, np.float32)


def _collect():
    import torch
    from audiomuse_ai_b200 import dist as amdist
    lib = _lib.load()
    _lib.check(lib.am_init(0))
    out = {}
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.profile_enable(True)
    for N, d, k in SHAPES:
        key = f"N{N}/d{d}/k{k}"
        x, init = _data(N, d, k, N + 7 * d + k)
        xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(init).cuda()
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        new = lambda: (torch.empty(N, dtype=torch.int32, device="cuda"), torch.empty(k, d, device="cuda"),  # noqa: E731
                       torch.empty(k, device="cuda"), torch.zeros(1, device="cuda"), torch.empty(N, device="cuda"))
        torch.cuda.synchronize()
        _kernels()
        lab, sums, cnt, inert, _ = new()
        _lib.check(lib.am_kmeans_assign_dev(p(xd), N, d, p(cd), k, p(lab), p(sums), p(cnt), p(inert), st))
        out.update({f"{key}/assign/labels": lab.cpu().numpy(), f"{key}/assign/counts": cnt.cpu().numpy(),
                    f"{key}/assign/sums": sums.cpu().numpy(), f"{key}/assign/inertia": inert.cpu().numpy(),
                    f"{key}/assign/kernels": _kernels()})
        plan = amdist.KMeansPlan(xd, k)
        lab, sums, cnt, inert, dist = new()
        plan.step(cd, lab, sums, cnt, inert, dist)
        lab2, _, _, inert2, _ = new()
        plan.step(cd, lab2, None, None, inert2)
        torch.cuda.synchronize()
        out.update({f"{key}/plan/tensor_cores": np.array(plan.uses_tensor_cores),
                    f"{key}/plan/labels": lab.cpu().numpy(), f"{key}/plan/counts": cnt.cpu().numpy(),
                    f"{key}/plan/dist": dist.cpu().numpy(), f"{key}/plan/sums": sums.cpu().numpy(),
                    f"{key}/plan/inertia": inert.cpu().numpy(), f"{key}/plan_inertia_only/labels": lab2.cpu().numpy(),
                    f"{key}/plan_inertia_only/inertia": inert2.cpu().numpy()})
        plan.close()
        out[f"{key}/plan/kernels"] = _kernels()
        for name, kw in (("fit_init", dict(init_centers=init)), ("fit_seeded", dict(n_init=2, seed=N + k))):
            c, lab, inertia, it = cg.kmeans_fit(x, k, max_iter=FIT_ITERS, **kw)
            out.update({f"{key}/{name}/centers": c, f"{key}/{name}/labels": lab,
                        f"{key}/{name}/inertia": np.array([inertia]), f"{key}/{name}/n_iter": np.array([it]),
                        f"{key}/{name}/kernels": _kernels()})
        print(f"{key}: tensor cores in plan={plan.uses_tensor_cores}", flush=True)
    _lib.profile_enable(False)
    return out


def _close(k, want, got):
    """None when `got` matches `want` as this array's kind requires, else a description of the difference."""
    kind = k.rsplit("/", 1)[1]
    if kind in ("kernels", "tensor_cores", "counts", "dist") or (kind == "labels" and "/fit_" not in k):
        return None if np.array_equal(want, got) else "not identical"
    if kind == "sums":
        return None if np.allclose(got, want, rtol=2e-5, atol=2e-3) else f"max |diff| {np.abs(got - want).max():.3g}"
    if kind == "inertia":
        rel = abs(float(got[0]) - float(want[0])) / max(abs(float(want[0])), 1e-30)
        return None if rel <= 1e-5 else f"relative {rel:.3g}"
    if kind == "labels":
        eq = float((got == want).mean())
        return None if eq > 0.999 else f"{eq:.5f} equal"
    if kind == "centers":
        err = float(np.abs(got - want).max())
        return None if err <= 1e-4 * max(1.0, float(np.abs(want).max())) else f"max |diff| {err:.3g}"
    if kind == "n_iter":
        return None if abs(int(got[0]) - int(want[0])) <= 1 else f"{int(want[0])} -> {int(got[0])}"
    return None if np.array_equal(want, got) else "not identical"


def _renumber(want, got):
    """A seeded fit's restarts may reach the same optimum with its clusters numbered differently, and float-atomic
    noise in the inertia decides which restart is kept: number got's clusters after want's nearest centres when that
    maps them one to one."""
    for k in [k for k in got if k.endswith("/centers") and k in want.files]:
        w, g = want[k], got[k]
        perm = ((g[:, None, :].astype(np.float64) - w[None, :, :]) ** 2).sum(2).argmin(1)
        if len(set(perm.tolist())) == len(perm):
            c = np.empty_like(g)
            c[perm] = g
            got[k], got[k[:-7] + "labels"] = c, perm[got[k[:-7] + "labels"]].astype(np.int32)


def main():
    mode, path = sys.argv[1], sys.argv[2]
    got = _collect()
    if mode == "dump":
        np.savez(path, **got)
        print(f"wrote {len(got)} arrays to {path}")
        return 0
    want = np.load(path)
    _renumber(want, got)
    bad = []
    for k in sorted(set(want.files) | set(got)):
        why = "missing on one side" if k not in got or k not in want.files else _close(k, want[k], got[k])
        if why:
            bad.append(k)
            print(f"DIFFERENT: {k}: {why}" + (f": {' '.join(want[k])} -> {' '.join(got[k])}"
                                               if k.endswith("kernels") and why == "not identical" else ""))
    exact = sum(1 for k in got if k in want.files and np.array_equal(want[k], got[k]))
    print(f"{len(got) - len(bad)} of {len(got)} arrays match ({exact} bit-identical), {len(bad)} different")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
