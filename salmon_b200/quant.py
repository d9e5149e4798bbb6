"""Host-side mirror of `salmon quant` for the hot path (src/quant/SalmonQuantify.cpp:2777-2956 ->
quantifyLibrary -> stageFinalizeMappingOutputs, src/quant/pipeline/MappingPipelineStages.cpp:37-206):

    reads --sb_map_batch--> per-read alignments, online masses / FLD, per-batch class tables
          --sb_map_finish--> equivalence classes (EquivalenceClassBuilder::finish) + normalizeAlphas
          --sb_em_optimize--> alpha (CollapsedEMOptimizer::optimize)
          --sb_tpm / sb_write_quant_sf / sb_write_eq_classes--> quant.sf, aux_info/eq_classes.txt.gz

One process per GPU; with torch.distributed initialised (world > 1) every rank maps its own read shard, the
end-of-mapping statistics are reduced once (salmon_b200.dist) and the EM all-reduces alpha per iteration (NCCL).
"""
from __future__ import annotations

import os

import numpy as np

from . import _capi
from ._capi import EMContext, EqClasses, MapContext, default_params, map_default_params


def _boot_params(ep):
    """the bootstrap replicates run with at least 50 iterations (CollapsedEMOptimizer.cpp:411), like sb_quant_files"""
    import copy
    bp = copy.copy(ep)
    bp.min_iter = 50
    return bp


def _em_options(ep, meta=False, alternative_init_mode=False, bootstrap_reproject=False):
    """salmon's offline-phase options on em_params (DESIGN.md section 15): `--alternativeInitMode`,
    `--bootstrapReproject`, then the `--meta` preset, which overrides the values given for the same options
    (QuantOptionsUtils.cpp:449-454); the defaults leave ep as it is"""
    if alternative_init_mode:
        ep.alt_init = 1
    if bootstrap_reproject:
        ep.bootstrap_reproject = 1
    if meta:
        ep.init_uniform = 1
        ep.no_rich_eq = 1
        ep.use_vbem = 0
        ep.alt_init = 1      # metaGenomeMode (CollapsedEMOptimizer.cpp:800-810): no effect beside initUniform
    return ep


def _likelihood_options(mp, incompat_prior, no_single_frag_prob, no_frag_len_dist, no_eff_len_correction):
    """salmon's fragment-likelihood options on map_params (DESIGN.md section 13); the defaults leave mp as it is"""
    if incompat_prior:
        p = float(incompat_prior)
        mp.incompat_prior = 0.0 if p < 1e-100 else p     # below 1e-100: incompatible mappings are ignored
    if no_single_frag_prob:
        mp.no_single_frag_prob = 1
    if no_frag_len_dist:
        mp.no_frag_len_dist = 1
    if no_eff_len_correction:
        mp.no_eff_len_correction = 1
    return mp


def _mimic_options(mp, min_aln_prob, mimic_bt2, mimic_strict_bt2):
    """`--minAlnProb`, then `--mimicBT2` / `--mimicStrictBT2` (sb_map_mimic_bt2, DESIGN.md section 14), which override
    the values given for the same options; the defaults leave mp as it is"""
    if mimic_bt2 and mimic_strict_bt2:
        raise _capi.SalmonB200Error("You passed both the --mimicBT2 and --mimicStrictBT2 parameters.  These are mutually "
                                    "exclusive. Please select only one of these flags.")
    if min_aln_prob is not None:
        if not 0.0 <= float(min_aln_prob) <= 1.0:
            raise _capi.SalmonB200Error(f"--minAlnProb takes a probability in [0, 1], got {min_aln_prob}")
        mp.min_aln_prob = float(min_aln_prob)
    if mimic_bt2 or mimic_strict_bt2:
        _capi.map_mimic_bt2(mp, strict=bool(mimic_strict_bt2))
    return mp


def _drop_decoys(index, inputs):
    """readExp.dropDecoyTranscripts() (SalmonQuantify.cpp:2479, ReadExperiment.hpp:120): decoys -- the suffix of the id
    space, never part of a label -- leave before the optimiser and the writers.  Returns (Mq, inputs cut to Mq)."""
    M = index.n_txps
    fd = index.meta()["first_decoy"]
    Mq = fd if fd < M else M
    if Mq == M:
        return M, inputs
    cut = dict(inputs)
    for k in ("projected_counts", "eff_len", "unique_counts", "total_counts"):
        if k in cut and cut[k] is not None:
            cut[k] = np.ascontiguousarray(cut[k][:Mq])
    return Mq, cut


def quant_reads(index, left, right, map_params=None, em_params=None, device=0, batch=262_144, dist=None,
                names=None, out_dir=None, dump_eq=False, dump_eq_weights=False, incompat_prior=0.0,
                no_single_frag_prob=False, no_frag_len_dist=False, no_eff_len_correction=False, min_aln_prob=None,
                mimic_bt2=False, mimic_strict_bt2=False):
    """left/right: [n, L] uint8 base codes (0..3 = ACGT, 4 = N) of THIS rank's read shard.  incompat_prior,
    no_single_frag_prob, no_frag_len_dist, no_eff_len_correction: `--incompatPrior`, `--noSingleFragProb`,
    `--noFragLengthDist`, `--noEffectiveLengthCorrection` (set on map_params; DESIGN.md section 13).  min_aln_prob,
    mimic_bt2, mimic_strict_bt2: `--minAlnProb`, `--mimicBT2`, `--mimicStrictBT2` (DESIGN.md section 14).
    Returns dict(alpha, tpm, eff_len, classes, n_mapped, em_stats)."""
    mp = _likelihood_options(map_params or map_default_params(), incompat_prior, no_single_frag_prob, no_frag_len_dist,
                             no_eff_len_correction)
    _mimic_options(mp, min_aln_prob, mimic_bt2, mimic_strict_bt2)
    ep = em_params or default_params()
    n, L = left.shape
    world = dist.get_world_size() if (dist is not None and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    ctx = MapContext(index, mp, device=device, batch_cap=min(batch, max(n, 1)), max_read_len=L)
    for s in range(0, n, batch):
        ctx.map_batch(left[s:s + batch], right[s:s + batch])
    res = ctx.finish()
    inputs = res
    n_mapped = res["counters"]["n_mapped"]
    if world > 1:
        from .dist import reduce_partials
        g, roots = reduce_partials(ctx.partial(), dist, f"cuda:{device}")
        inputs = ctx.project_global(g, roots)
        n_mapped = g["assigned"]
    ctx.close()
    M, inputs = _drop_decoys(index, inputs)
    eq = EqClasses(M, res["off"], res["tids"], res["weights"], res["counts"])
    em = EMContext(device)
    if world > 1:
        em.peer_setup(dist, M)          # alpha all-reduced inside the persistent kernel over NVLink peer memory
    alpha, st, ok = em.optimize(eq, ep, inputs["projected_counts"], inputs["eff_len"], inputs["unique_counts"])
    em.close()
    if not ok:
        raise _capi.SalmonB200Error("The optimization algorithm failed (total alpha weight too small)")
    tpm = _capi.tpm(alpha, inputs["eff_len"], float(n_mapped) if n_mapped else None)
    if out_dir is not None and rank == 0:
        os.makedirs(os.path.join(out_dir, "aux_info"), exist_ok=True)
        nm = names or [f"t{i}" for i in range(M)]
        meta = index.meta()
        if names is None and meta["names"]:
            nm = meta["names"]
        nm = nm[:M]
        lens = (meta["complete_len"] if meta["complete_len"] is not None else index.tx_lengths())[:M]
        _capi.write_quant_sf(os.path.join(out_dir, "quant.sf"), nm, lens, inputs["eff_len"], alpha,
                             float(n_mapped) if n_mapped else None)
        if dump_eq or dump_eq_weights:
            _capi.write_eq_classes(os.path.join(out_dir, "aux_info", "eq_classes.txt.gz"), nm, res["off"], res["tids"],
                                   res["counts"], res["weights"] if dump_eq_weights else None)
    return dict(alpha=alpha, tpm=tpm, eff_len=inputs["eff_len"], classes=res, n_mapped=int(n_mapped), em_stats=st,
                projected_counts=inputs["projected_counts"], unique_counts=inputs["unique_counts"])


def _quantify(index, ctx, ep, device, dist, names, out_dir, dump_eq, dump_eq_weights, num_bootstraps=0, seed=0,
              n_observed=None, skip_quant=False):
    """Everything after mapping: finish() -> (multi-GPU reduction) -> EM -> outputs.  Shared by quant_reads-style
    callers that drive the MapContext themselves."""
    world = dist.get_world_size() if (dist is not None and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    if skip_quant:
        return _skip_quant(index, ctx, device, dist, names, out_dir, dump_eq, dump_eq_weights, ep, n_observed)
    res = ctx.finish()
    inputs = res
    n_mapped = res["counters"]["n_mapped"]
    if world > 1:
        from .dist import reduce_partials
        g, roots = reduce_partials(ctx.partial(), dist, f"cuda:{device}")
        inputs = ctx.project_global(g, roots)
        n_mapped = g["assigned"]
    ctx.close()
    M, inputs = _drop_decoys(index, inputs)
    eq = EqClasses(M, res["off"], res["tids"], res["weights"], res["counts"])
    em = EMContext(device)
    if world > 1:
        em.peer_setup(dist, M)
    alpha, st, ok = em.optimize(eq, ep, inputs["projected_counts"], inputs["eff_len"], inputs["unique_counts"])
    if not ok:
        em.close()
        raise _capi.SalmonB200Error("The optimization algorithm failed (total alpha weight too small)")
    boots = None
    if num_bootstraps > 0 and world == 1:
        boots, _ = em.bootstrap(_boot_params(ep), float(n_mapped), num_bootstraps, seed)
    em.close()
    tpm = _capi.tpm(alpha, inputs["eff_len"], float(n_mapped) if n_mapped else None)
    if out_dir is not None and rank == 0:
        os.makedirs(os.path.join(out_dir, "aux_info"), exist_ok=True)
        meta = index.meta()
        nm = (names or meta["names"] or [f"t{i}" for i in range(index.n_txps)])[:M]
        lens = (meta["complete_len"] if meta["complete_len"] is not None else index.tx_lengths())[:M]
        _capi.write_quant_sf(os.path.join(out_dir, "quant.sf"), nm, lens, inputs["eff_len"], alpha,
                             float(n_mapped) if n_mapped else None)
        if dump_eq or dump_eq_weights:
            _capi.write_eq_classes(os.path.join(out_dir, "aux_info", "eq_classes.txt.gz"), nm, res["off"], res["tids"],
                                   res["counts"], res["weights"] if dump_eq_weights else None)
        if boots is not None:
            os.makedirs(os.path.join(out_dir, "aux_info", "bootstrap"), exist_ok=True)
            w = _capi.BootstrapWriter(os.path.join(out_dir, "aux_info", "bootstrap", "bootstraps.gz"))
            for b in boots:
                w.write(b)
            w.close()
    return dict(alpha=alpha, tpm=tpm, eff_len=inputs["eff_len"], classes=res, n_mapped=int(n_mapped), em_stats=st,
                projected_counts=inputs["projected_counts"], unique_counts=inputs["unique_counts"], bootstraps=boots,
                n_observed=n_observed)


def _skip_quant(index, ctx, device, dist, names, out_dir, dump_eq, dump_eq_weights, ep, n_observed):
    """`--skipQuant` (MappingPipelineStages.cpp:45-162): the classes without normalizeAlphas' projection, no optimiser,
    no quant.sf, no samples; under dump_eq_weights the dumped weights are the combined weights, computed on the device
    (sb_eq_combined_weights)"""
    world = dist.get_world_size() if (dist is not None and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    ctx.set_option("no_projection", 1)
    res = ctx.finish()
    inputs = res
    n_mapped = res["counters"]["n_mapped"]
    if world > 1:
        from .dist import reduce_partials
        g, roots = reduce_partials(ctx.partial(), dist, f"cuda:{device}")
        inputs = ctx.project_global(g, roots)
        n_mapped = g["assigned"]
    ctx.close()
    M, inputs = _drop_decoys(index, inputs)
    combined = None
    if dump_eq_weights:
        em = EMContext(device)
        combined = em.combined_weights(EqClasses(M, res["off"], res["tids"], res["weights"], res["counts"]),
                                       inputs["eff_len"], no_rich_eq=bool(ep.no_rich_eq))
        em.close()
    if out_dir is not None and rank == 0 and (dump_eq or dump_eq_weights):
        os.makedirs(os.path.join(out_dir, "aux_info"), exist_ok=True)
        meta = index.meta()
        nm = (names or meta["names"] or [f"t{i}" for i in range(index.n_txps)])[:M]
        _capi.write_eq_classes(os.path.join(out_dir, "aux_info", "eq_classes.txt.gz"), nm, res["off"], res["tids"],
                               res["counts"], combined)
    return dict(alpha=None, tpm=None, eff_len=inputs["eff_len"], classes=res, n_mapped=int(n_mapped), em_stats=None,
                projected_counts=None, unique_counts=inputs["unique_counts"], bootstraps=None, n_observed=n_observed,
                combined_weights=combined)


def quant_files(index, mates1, mates2, out_dir=None, map_params=None, em_params=None, device=0, batch=262_144,
                max_read_len=256, threads=8, dist=None, dump_eq=False, dump_eq_weights=False, num_bootstraps=0, seed=0,
                write_mappings=None, write_qualities=False, write_unmapped_names=False, cmdline="", recover_orphans=False,
                softclip=0, incompat_prior=0.0, no_single_frag_prob=False, no_frag_len_dist=False,
                no_eff_len_correction=False, min_aln_prob=None, mimic_bt2=False, mimic_strict_bt2=False,
                skip_quant=False, bootstrap_reproject=False, meta=False, alternative_init_mode=False):
    """`salmon quant -i index -l IU -1 mates1 -2 mates2 -o out_dir` for the hot path: FASTQ/FASTA(.gz) files ->
    sb_reads_bucketed -> sb_map_batch -> ... -> quant.sf.  index: an _capi.Index or the path of a saved one.  With
    torch.distributed initialised every rank takes the global batches g with g % world == rank (round-robin sharding
    of the read stream, SURVEY.md 8e), the end-of-mapping statistics are reduced once and the EM all-reduces alpha.
    A pair whose mates differ in length is mapped at the shorter length (documented deviation until the kernels take
    per-mate lengths).  write_mappings: path of a SAM file of the mappings (`--writeMappings=FILE`), with the reads'
    qualities when write_qualities; write_unmapped_names: out_dir/aux_info/unmapped_names.txt.  Both need one GPU.
    recover_orphans: `--recoverOrphans` (sets map_params.recover_orphans; single-end reads: no effect).
    softclip: scoring mode of the DP (sets map_params.softclip when non-zero): 1 = `--softclipOverhangs`, 2 =
    `--softclip` (DESIGN.md section 12).  incompat_prior, no_single_frag_prob, no_frag_len_dist, no_eff_len_correction:
    `--incompatPrior`, `--noSingleFragProb`, `--noFragLengthDist`, `--noEffectiveLengthCorrection` (DESIGN.md section
    13).  min_aln_prob, mimic_bt2, mimic_strict_bt2: `--minAlnProb`, `--mimicBT2`, `--mimicStrictBT2`, applied after the
    other options so that the presets override them (DESIGN.md section 14).  skip_quant, bootstrap_reproject, meta,
    alternative_init_mode: `--skipQuant`, `--bootstrapReproject`, `--meta`, `--alternativeInitMode` (DESIGN.md section
    15); with skip_quant the result has no alpha and, under dump_eq_weights, the combined weights."""
    if isinstance(index, (str, bytes, os.PathLike)):
        index = _capi.Index.load(index)
    mp = map_params or map_default_params()
    if recover_orphans:
        mp.recover_orphans = 1
    if softclip:
        mp.softclip = int(softclip)
    _likelihood_options(mp, incompat_prior, no_single_frag_prob, no_frag_len_dist, no_eff_len_correction)
    _mimic_options(mp, min_aln_prob, mimic_bt2, mimic_strict_bt2)
    first_decoy = index.meta()["first_decoy"]
    if first_decoy < index.n_txps:
        mp.first_decoy = first_decoy
    ep = _em_options(em_params or default_params(), meta, alternative_init_mode, bootstrap_reproject)
    world = dist.get_world_size() if (dist is not None and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    ctx = MapContext(index, mp, device=device, batch_cap=batch, max_read_len=max_read_len)
    # sb_reads_bucketed: a reader thread parses and groups the reads by length into page-locked [n, L] buffers while this
    # thread maps the previous ones; global batches of `batch` records go round-robin to the ranks
    def map_one(left, right, L):
        ctx.map_batch(left, right)       # raises on error (the reader then stops and reports it)
        return 0
    if write_mappings or write_unmapped_names:
        if world > 1:
            raise _capi.SalmonB200Error("write_mappings / write_unmapped_names are written by a one-GPU run only: a "
                                        "read-sharded run cannot write them")
        un = None
        if write_unmapped_names:
            if out_dir is None:
                raise _capi.SalmonB200Error("write_unmapped_names needs an output directory")
            os.makedirs(os.path.join(out_dir, "aux_info"), exist_ok=True)
            un = os.path.join(out_dir, "aux_info", "unmapped_names.txt")
        sink = _capi.SamSink(index, write_mappings, un, cmdline=cmdline, qualities=write_qualities)
        try:
            ctx.attach_sam(sink)

            def map_sam(left, right, L, names, ql, qr):
                ctx.map_batch_sam(left, right, names, (ql, qr) if write_qualities else None)
                return 0
            with _capi.ReadFiles(mates1, mates2, n_threads=threads) as rf:
                st, dropped = rf.bucketed_meta(map_sam, min_len=mp.k, batch=batch, max_read_len=max_read_len,
                                               threads=threads, quals=write_qualities)
            if dropped:
                sink.write_unmapped(b"".join(nm + b" u\n" for nm in dropped))
            ctx.attach_sam(None)
        finally:
            sink.close()
    else:
        with _capi.ReadFiles(mates1, mates2, n_threads=threads) as rf:
            st = rf.bucketed(map_one, min_len=mp.k, batch=batch, max_read_len=max_read_len, threads=threads,
                             shard_index=rank, shard_count=world)
    n_observed = int(st["n_observed"])
    return _quantify(index, ctx, ep, device, dist, None, out_dir, dump_eq, dump_eq_weights, num_bootstraps, seed,
                     n_observed=n_observed, skip_quant=skip_quant)


def quant_eqclasses(eq_path, out_dir=None, em_params=None, device=0, num_bootstraps=0, seed=0,
                    bootstrap_reproject=False, meta=False, alternative_init_mode=False):
    """`salmon quant --eqclasses eq_classes.txt[.gz]` (EM only; src/quant/SalmonQuantify.cpp eq-class mode ->
    CollapsedEMOptimizer::optimize with eq_class_mode): BASELINE.json configs[1].  bootstrap_reproject, meta,
    alternative_init_mode: `--bootstrapReproject`, `--meta`, `--alternativeInitMode` (DESIGN.md section 15)."""
    f = _capi.read_eq_classes(eq_path)
    if not f["has_weights"]:
        raise _capi.SalmonB200Error("--eqclasses input needs the weights (write it with --dumpEqWeights)")
    M = f["n_txps"]
    eq = EqClasses(M, f["off"], f["tids"], f["weights"], f["counts"])
    # processEqClasses (src/alignment/SalmonQuantifyAlignments.cpp:1406-1440): fresh transcripts (no projected counts,
    # no unique counts), initUniform + eqClassMode, effective lengths taken from the file as they are
    projected = np.zeros(M)
    uniq = np.zeros(M, dtype=np.uint64)
    ep = _em_options(em_params or default_params(), meta, alternative_init_mode, bootstrap_reproject)
    ep.eq_class_mode = 1
    ep.init_uniform = 1
    em = EMContext(device)
    alpha, st, ok = em.optimize(eq, ep, projected, f["eff_len"], uniq)
    if not ok:
        em.close()
        raise _capi.SalmonB200Error("The optimization algorithm failed (total alpha weight too small)")
    n_frags = float(f["counts"].sum())
    boots = None
    if num_bootstraps > 0:
        boots, _ = em.bootstrap(_boot_params(ep), n_frags, num_bootstraps, seed)
    em.close()
    tpm = _capi.tpm(alpha, f["eff_len"], n_frags)
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        lens = np.maximum(f["eff_len"], 1).astype(np.uint32)   # the eq file carries no transcript lengths
        _capi.write_quant_sf(os.path.join(out_dir, "quant.sf"), f["names"], lens, f["eff_len"], alpha, n_frags)
    return dict(alpha=alpha, tpm=tpm, eff_len=f["eff_len"], em_stats=st, names=f["names"], bootstraps=boots)
