"""One process per GPU over torch.distributed (NCCL on GPU machines, gloo in CPU tests).

SURVEY 8(e): tracks are independent, so analysis shards a contiguous block of the sorted track
list per rank with NO data-path collective; afterwards ONE all-gather of the f32[N/W, 512]
embedding shards lands the full library matrix on every rank (k-NN then runs on a replicated
index with queries sharded round-robin: no further communication).  k-means keeps rows sharded
and all-reduces the [k, d] partial sums + [k] counts once per Lloyd iteration.

PyTorch is plumbing only here (device buffers, streams, the process group); the arithmetic is
libaudiomuse_b200's, called through device pointers.
"""
from __future__ import annotations

import os
from typing import Tuple

import numpy as np


def env_world() -> Tuple[int, int, int]:
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)),
            int(os.environ.get("WORLD_SIZE", 1)))


def shard_bounds(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of rank ``rank``: sizes differ by at most one, earlier ranks larger."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def padded_shard_len(n_items: int, world: int) -> int:
    return (n_items + world - 1) // world


def init_process_group(backend: str | None = None):
    import torch
    import torch.distributed as dist

    rank, local_rank, world = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    elif torch.cuda.is_available():
        torch.cuda.set_device(local_rank)
    return rank, local_rank, world


def bind_to_gpu_numa_node(local_rank: int):
    """Pin this process (and therefore the pinned host buffers it allocates next: first touch) to the CPU cores of the
    NUMA node its GPU hangs off.  With one process per GPU and ~250 MB of PCM copied host->device per step, ranks left on
    a remote socket share one inter-socket link (8 ranks: end-to-end efficiency 0.90 vs 0.99 device-resident).
    Best effort: returns the node id, or None when the topology cannot be read (no sysfs, one node, no permission)."""
    try:
        import torch
        prop = torch.cuda.get_device_properties(local_rank)
        bdf = f"{getattr(prop, 'pci_domain_id', 0):04x}:{prop.pci_bus_id:02x}:{prop.pci_device_id:02x}.0"
        base = f"/sys/bus/pci/devices/{bdf}"
        with open(f"{base}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            spec = f.read().strip()
        cpus = set()
        for part in spec.split(","):
            if "-" in part:
                a, b = part.split("-")
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        allowed = os.sched_getaffinity(0)
        cpus &= allowed
        if not cpus or cpus == allowed:
            return node if cpus else None
        os.sched_setaffinity(0, cpus)
        return node
    except Exception:
        return None


def all_gather_embeddings(local, n_total: int):
    """local: torch tensor [n_local, d] (this rank's shard, rows in shard_bounds order)
    -> [n_total, d] on every rank.  Shards are padded to equal length for the collective and
    the padding is dropped afterwards (SURVEY 8(e): "pad last shard to equal counts")."""
    import torch
    import torch.distributed as dist

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local[:n_total]
    world, rank = dist.get_world_size(), dist.get_rank()
    d = local.shape[1]
    plen = padded_shard_len(n_total, world)
    buf = torch.zeros((plen, d), dtype=local.dtype, device=local.device)
    buf[: local.shape[0]] = local
    full = torch.empty((world * plen, d), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(full, buf)
    parts = []
    for r in range(world):
        lo, hi = shard_bounds(n_total, r, world)
        parts.append(full[r * plen : r * plen + (hi - lo)])
    return torch.cat(parts, dim=0)


def all_reduce_sum_(*tensors):
    import torch.distributed as dist

    if dist.is_initialized() and dist.get_world_size() > 1:
        for t in tensors:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)


def max_over_ranks(value: float, device=None) -> float:
    import torch
    import torch.distributed as dist

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device=None) -> float:
    import torch
    import torch.distributed as dist

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def _relocate_empty_clusters(x_local, labels, centers, sums, counts):
    """sklearn's empty-cluster rule on sharded rows (same as am_kmeans_fit, kmeans.cu relocate_empty_kernel):
    the i-th empty cluster takes the point that is i-th farthest from its own centre; that row leaves the sums /
    counts of its donor cluster.  Each rank offers its farthest rows, one all-gather picks the global ones, and
    every rank applies the same sequential edits to its replicated sums / counts.  No-op without empty clusters."""
    import torch
    import torch.distributed as dist

    empty = torch.nonzero(counts == 0).flatten()
    m = int(empty.numel())
    if m == 0:
        return
    n_local, d = x_local.shape
    far = torch.empty((n_local,), dtype=torch.float32, device=x_local.device)
    for b0 in range(0, n_local, 65536):  # distances to the assigned centres, in row blocks
        xb = x_local[b0:b0 + 65536]
        far[b0:b0 + 65536] = ((xb - centers[labels[b0:b0 + 65536].long()]) ** 2).sum(1)
    kk = min(m, n_local)
    cand = torch.full((m, d + 2), -1.0, dtype=torch.float32, device=x_local.device)
    if kk > 0:
        vals, idx = torch.topk(far, kk)
        cand[:kk, 0] = vals
        cand[:kk, 1] = labels[idx].float()
        cand[:kk, 2:] = x_local[idx]
    if dist.is_initialized() and dist.get_world_size() > 1:
        full = torch.empty((dist.get_world_size() * m, d + 2), dtype=torch.float32, device=x_local.device)
        dist.all_gather_into_tensor(full, cand)
        cand = full
    order = torch.sort(cand[:, 0], descending=True, stable=True).indices[:m]
    for e in range(m):
        row = cand[order[e]]
        if float(row[0]) < 0:  # fewer rows than empty clusters
            break
        donor, target = int(row[1].item()), int(empty[e].item())
        sums[donor] -= row[2:]
        sums[target] = row[2:]
        counts[target] = 1.0
        counts[donor] -= 1.0


class KMeansPlan:
    """am_kmeans_plan over this rank's rows (torch.cuda f32[n_local, d]): the split-bf16 copy is built once, every
    step is one tensor-core assignment pass + one partial-sum pass, stream-ordered on torch's current stream.
    The rows are expected centred (column means near 0): both steps decide on fp32 ||c||^2 - 2 x.c, whose
    cancellation grows with ||x||^2.  am_kmeans_fit centres its copy of the rows itself."""

    def __init__(self, x_local, k: int):
        import ctypes as C

        import torch

        from . import _lib

        self._lib = _lib.load()
        self._check = _lib.check
        self.x = x_local.contiguous()
        self.k = int(k)
        h = C.c_void_p()
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self._check(self._lib.am_kmeans_plan_create(self.x.data_ptr(), self.x.shape[0], self.x.shape[1], self.k, st, C.byref(h)))
        self._h = h
        self.uses_tensor_cores = bool(self._lib.am_kmeans_plan_uses_tensor_cores(h))

    def step(self, centers, labels, sums=None, counts=None, inertia=None, dist=None):
        import ctypes as C

        import torch

        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        self._check(self._lib.am_kmeans_plan_step(self._h, p(centers), p(labels), p(sums), p(counts), p(inertia), p(dist),
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def last_recheck(self) -> int:
        """rows the last step re-checked in exact fp32 (near-ties inside the tensor-core error band)"""
        import ctypes as C

        import torch

        n = C.c_int(0)
        self._check(self._lib.am_kmeans_plan_last_recheck(self._h, C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(n)))
        return int(n.value)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.am_kmeans_plan_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def kmeans_lloyd_sharded(x_local, centers, max_iter=300, tol=1e-4, timing=None):
    """Multi-GPU Lloyd: x_local torch.cuda f32[n_local, d] (this rank's rows), centers torch.cuda
    f32[k, d] replicated.  Per iteration: one am_kmeans_plan_step on the shard, then one all-reduce of
    the [k, d] sums and [k] counts (the only collective; + one scalar for the inertia at the end).
    tol=None runs exactly max_iter iterations without the convergence read-back (timing runs).
    `timing`, when a dict, receives {"assign_ms", "allreduce_ms"} device times summed over the iterations.
    The rows are expected centred, as for KMeansPlan.  Returns (centers, labels_local, inertia, n_iter)."""
    import torch

    n_local, d = x_local.shape
    k = centers.shape[0]
    centers = centers.clone().contiguous()
    labels = torch.empty((n_local,), dtype=torch.int32, device=x_local.device)
    sums = torch.empty((k, d), dtype=torch.float32, device=x_local.device)
    counts = torch.empty((k,), dtype=torch.float32, device=x_local.device)
    inertia = torch.zeros((1,), dtype=torch.float32, device=x_local.device)
    var_mean = 0.0
    if tol is not None:
        # tolerance scaled by the mean feature variance over the WHOLE data set (sklearn rule)
        s1 = x_local.sum(0, dtype=torch.float64)
        s2 = (x_local.double() ** 2).sum(0)
        n = torch.tensor([float(n_local)], dtype=torch.float64, device=x_local.device)
        all_reduce_sum_(s1, s2, n)
        var_mean = float(((s2 / n) - (s1 / n) ** 2).mean().item())
    plan = KMeansPlan(x_local, k)
    ev = []
    it = 0
    try:
        for it in range(1, max_iter + 1):
            if timing is not None:
                e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                e[0].record()
            plan.step(centers, labels, sums, counts)
            if timing is not None:
                e[1].record()
            all_reduce_sum_(sums, counts)
            if timing is not None:
                e[2].record()
                ev.append(e)
            if tol is not None:
                _relocate_empty_clusters(x_local, labels, centers, sums, counts)
            new_centers = torch.where(counts[:, None] > 0, sums / counts.clamp(min=1.0)[:, None], centers)
            if tol is not None:
                shift = float(((new_centers - centers).double() ** 2).sum().item())
            centers = new_centers.contiguous()
            if tol is not None and shift <= tol * var_mean:
                break
        plan.step(centers, labels, None, None, inertia)
        all_reduce_sum_(inertia)
        result = float(inertia.item())
        if timing is not None:
            timing["assign_ms"] = sum(a.elapsed_time(b) for a, b, _ in ev)
            timing["allreduce_ms"] = sum(b.elapsed_time(c) for _, b, c in ev)
            timing["tensor_cores"] = plan.uses_tensor_cores
    finally:
        plan.close()
    return centers, labels, result, it


def sharded_knn_query(index, queries, k: int):
    """SURVEY 8(e): the library is replicated (after the all-gather), the QUERIES are sharded round-robin over the
    ranks; each rank answers its share on its own GPU and one all-gather of the [nq/W, k] (id, distance) pairs puts
    the complete answer on every rank.  index: voyager_compat.Index (same contents on every rank);
    queries: numpy f32[nq, d] (same on every rank).  Returns (ids i64[nq, k], dist f32[nq, k])."""
    import torch
    import torch.distributed as dist

    queries = np.ascontiguousarray(queries, dtype=np.float32)
    nq = queries.shape[0]
    if not dist.is_initialized() or dist.get_world_size() == 1:
        ids, dd = index.query(queries, k)
        return np.asarray(ids, dtype=np.int64), np.asarray(dd, dtype=np.float32)
    world, rank = dist.get_world_size(), dist.get_rank()
    mine = queries[rank::world]
    per = (nq + world - 1) // world
    ids_l = np.full((per, k), -1, dtype=np.int64)
    dd_l = np.full((per, k), np.inf, dtype=np.float32)
    if len(mine):
        a, b = index.query(mine, k)
        ids_l[: len(mine)] = np.asarray(a, dtype=np.int64)
        dd_l[: len(mine)] = np.asarray(b, dtype=np.float32)
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    ti, td = torch.from_numpy(ids_l).to(dev), torch.from_numpy(dd_l).to(dev)
    gi = torch.empty((world * per, k), dtype=torch.int64, device=dev)
    gd = torch.empty((world * per, k), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(gi, ti)
    dist.all_gather_into_tensor(gd, td)
    gi, gd = gi.cpu().numpy().reshape(world, per, k), gd.cpu().numpy().reshape(world, per, k)
    ids = np.empty((nq, k), dtype=np.int64)
    dd = np.empty((nq, k), dtype=np.float32)
    for r in range(world):
        n_r = len(range(r, nq, world))
        ids[r::world] = gi[r, :n_r]
        dd[r::world] = gd[r, :n_r]
    return ids, dd
