"""Host layer of the multi-GPU path (SURVEY.md section 8e): one process per GPU, reads sharded over the ranks,
every rank keeps the equivalence classes of its own shard.  The only data-path collective is the per-iteration
all-reduce of alpha inside the EM (NCCL, in the library); what normalizeAlphas needs globally at the END of mapping
(M-sized vectors: masses, FLD, counts, cluster roots) is reduced once here, through torch.distributed (NCCL on the
GPU box, gloo in the CPU tests)."""
from __future__ import annotations

import numpy as np


def _t(x, device):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to(device)


def reduce_partials(p: dict, dist=None, device="cpu"):
    """p: MapContext.partial() of this rank.  Returns (global statistics dict, roots_all [world, M]).

    masses / FLD: sums in linear space (log-sum-exp over ranks; every rank's FLD contains the prior once, so the
    prior is subtracted world-1 times); counts: sums; fld_min: min; cluster roots: all-gathered (the union of the
    per-rank partitions is formed on the device by sb_map_project_global)."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return dict(p), p["cluster_root"][None, :].copy()
    import torch
    world = dist.get_world_size()

    def allreduce(x, op):
        t = _t(x, device)
        dist.all_reduce(t, op=op)
        return t.cpu().numpy()

    def lse(vals, prior=None):
        """log(sum_r exp(vals_r) - (world-1) * exp(prior)); +inf entries mean 'no mass' (salmon's LOG_0)."""
        v = np.where(np.isfinite(vals), vals, -np.inf)
        ref = allreduce(np.array([v.max() if v.size else -np.inf]), dist.ReduceOp.MAX)[0]
        if not np.isfinite(ref):
            return vals.copy()
        lin = np.exp(v - ref)
        if prior is not None:
            lin = np.maximum(lin - np.exp(prior - ref), 0.0)
        tot = allreduce(lin, dist.ReduceOp.SUM)
        if prior is not None:
            tot = tot + np.exp(prior - ref)
        with np.errstate(divide="ignore"):
            out = ref + np.log(tot)
        return np.where(tot > 0, out, np.inf)

    g = dict(p)
    g["mass"] = lse(p["mass"])
    g["fld_hist"] = lse(p["fld_hist"], p["fld_prior_hist"])
    g["fld_tot"] = float(lse(np.array([p["fld_tot"]]), np.array([p["fld_prior_tot"]]))[0])
    for k in ("unique_counts", "total_counts", "cluster_hits"):
        g[k] = allreduce(p[k].astype(np.int64), dist.ReduceOp.SUM).astype(np.uint64)
    g["fld_min"] = int(allreduce(np.array([p["fld_min"]], dtype=np.int64), dist.ReduceOp.MIN)[0])
    g["assigned"] = int(allreduce(np.array([p["assigned"]], dtype=np.int64), dist.ReduceOp.SUM)[0])
    g["compatible"] = int(allreduce(np.array([p.get("compatible", 0)], dtype=np.int64), dist.ReduceOp.SUM)[0])
    mine = _t(p["cluster_root"].astype(np.int64), device)
    parts = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine)
    roots_all = np.stack([q.cpu().numpy().astype(np.uint32) for q in parts])
    return g, roots_all
