"""ctypes binding of oracle/liboracle.so -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "liboracle.so")


class orc_em_params(C.Structure):
    _fields_ = [
        ("use_vbem", C.c_int32), ("per_txp_prior", C.c_int32), ("init_uniform", C.c_int32),
        ("eq_class_mode", C.c_int32), ("no_rich_eq", C.c_int32), ("no_length_correction", C.c_int32),
        ("alt_init", C.c_int32), ("n_threads", C.c_int32),
        ("vb_prior", C.c_double), ("tol", C.c_double), ("num_required_frags", C.c_double),
        ("min_iter", C.c_uint32), ("max_iter", C.c_uint32),
    ]


class orc_em_stats(C.Structure):
    _fields_ = [
        ("iters", C.c_uint32), ("converged", C.c_uint32), ("max_rel_diff", C.c_double),
        ("alpha_sum", C.c_double), ("n_degenerate", C.c_uint64), ("ok", C.c_int32),
    ]


_lib = None


def build():
    subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        lib = C.CDLL(LIB)
        lib.orc_digamma.restype = C.c_double
        lib.orc_digamma.argtypes = [C.c_double]
        # The C default is the platform libm (what the reference's std::exp / std::log are).  The regression tests demand
        # bit-exact labels / integer accumulators from the CUDA path, so the harness switches the oracle to its fdlibm
        # restatement (oracle/orc_math.h: the ALGORITHM the device code implements); the pinning tests
        # (tests/test_math_pinning.py, tests/test_map_gpu.py::test_gpu_vs_libm_oracle_at_scale) switch back with
        # math_mode("libm") and account for every label that differs.
        lib.orc_set_math_mode(1)
        _lib = lib
    return _lib


class math_mode:
    """with math_mode("libm"): ...  -- exp / log of the Stage A oracle for the duration of the block"""

    def __init__(self, mode):
        self.mode = {"libm": 0, "fdlibm": 1}[mode]

    def __enter__(self):
        lib = load()
        self.prev = lib.orc_get_math_mode()
        lib.orc_set_math_mode(self.mode)
        return self

    def __exit__(self, *a):
        load().orc_set_math_mode(self.prev)


def params_from(p, n_threads=0) -> orc_em_params:
    """Copy the shared fields of an sb_em_params (or dict) into orc_em_params."""
    o = orc_em_params()
    for k in ("use_vbem", "per_txp_prior", "init_uniform", "eq_class_mode", "no_rich_eq",
              "no_length_correction", "alt_init", "vb_prior", "tol", "num_required_frags",
              "min_iter", "max_iter"):
        setattr(o, k, p[k] if isinstance(p, dict) else getattr(p, k))
    o.n_threads = n_threads
    return o


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def em_optimize(eq, projected, eff_len, unique, p, mt=False, n_threads=0, want_combined=False):
    lib = load()
    M = eq.n_txps
    op = params_from(p, n_threads)
    alpha = np.empty(M, dtype=np.float64)
    st = orc_em_stats()
    projected = np.ascontiguousarray(projected, dtype=np.float64)
    eff_len = np.ascontiguousarray(eff_len, dtype=np.float64)
    unique = np.ascontiguousarray(unique, dtype=np.uint64)
    if mt:
        rc = lib.orc_em_optimize_mt(C.c_uint64(eq.n_classes), C.c_uint32(M), _p(eq.off), _p(eq.tids),
                                    _p(eq.weights), _p(eq.counts), _p(projected), _p(eff_len),
                                    _p(unique), C.byref(op), _p(alpha), C.byref(st))
        assert rc == 0
        return alpha, st
    cw = np.empty(eq.nnz, dtype=np.float64) if want_combined else None
    valid = np.empty(eq.n_classes, dtype=np.uint8) if want_combined else None
    rc = lib.orc_em_optimize(C.c_uint64(eq.n_classes), C.c_uint32(M), _p(eq.off), _p(eq.tids),
                             _p(eq.weights), _p(eq.counts), _p(projected), _p(eff_len), _p(unique),
                             C.byref(op), _p(alpha), _p(cw), _p(valid), None, C.byref(st))
    assert rc == 0
    if want_combined:
        return alpha, st, cw, valid
    return alpha, st


def em_step(eq, cw, valid, prior, alpha_in, vbem, serial=False, alpha_out_init=None):
    lib = load()
    M = eq.n_txps
    out = np.zeros(M) if alpha_out_init is None else np.array(alpha_out_init, dtype=np.float64)
    th = np.zeros(M)
    fn = lib.orc_em_step_serial if serial else lib.orc_em_step
    fn(C.c_uint64(eq.n_classes), C.c_uint32(M), _p(eq.off), _p(eq.tids), _p(np.ascontiguousarray(cw)),
       _p(eq.counts), _p(valid), _p(np.ascontiguousarray(prior, dtype=np.float64)),
       _p(np.ascontiguousarray(alpha_in, dtype=np.float64)), _p(out), _p(th), C.c_int(vbem))
    return out, th


def tpm(alpha, eff_len):
    lib = load()
    out = np.empty_like(alpha)
    lib.orc_tpm(C.c_uint32(alpha.shape[0]), _p(np.ascontiguousarray(alpha)),
                _p(np.ascontiguousarray(eff_len, dtype=np.float64)), _p(out))
    return out


def digamma(x):
    return load().orc_digamma(float(x))


def philox(c, k):
    out = (C.c_uint32 * 4)()
    load().orc_philox4x32(C.c_uint32(c[0]), C.c_uint32(c[1]), C.c_uint32(c[2]), C.c_uint32(c[3]),
                          C.c_uint32(k[0]), C.c_uint32(k[1]), out)
    return list(out)


def bootstrap(eq, cw, valid, prior, active, p, n_boot, seed):
    """orc_bootstrap -> (alphas [n_boot, M], sampled counts [n_boot, C], rc)."""
    lib = load()
    M, Cn = eq.n_txps, eq.n_classes
    op = params_from(p)
    alphas = np.zeros((n_boot, M))
    samp = np.zeros((n_boot, Cn), dtype=np.uint64)
    rc = lib.orc_bootstrap(C.c_uint64(Cn), C.c_uint32(M), _p(eq.off), _p(eq.tids), _p(np.ascontiguousarray(cw)),
                           _p(eq.counts), _p(np.ascontiguousarray(valid, dtype=np.uint8)),
                           _p(np.ascontiguousarray(prior, dtype=np.float64)),
                           _p(np.ascontiguousarray(active, dtype=np.uint8)), C.byref(op), C.c_uint32(n_boot),
                           C.c_uint64(seed), _p(alphas), _p(samp))
    return alphas, samp, rc


def gibbs(eq, valid, eff_len, alphas_init, use_vbem, per_txp_prior, vb_prior, n_samples, thinning, no_gamma_draw,
          num_mapped_frags, seed):
    lib = load()
    M = eq.n_txps
    out = np.zeros((n_samples, M))
    rc = lib.orc_gibbs(C.c_uint64(eq.n_classes), C.c_uint32(M), _p(eq.off), _p(eq.tids), _p(eq.weights),
                       _p(eq.counts), _p(np.ascontiguousarray(valid, dtype=np.uint8)),
                       _p(np.ascontiguousarray(eff_len, dtype=np.float64)),
                       _p(np.ascontiguousarray(alphas_init, dtype=np.float64)), C.c_int(use_vbem),
                       C.c_int(per_txp_prior), C.c_double(vb_prior), C.c_uint32(n_samples), C.c_uint32(thinning),
                       C.c_int(no_gamma_draw), C.c_double(num_mapped_frags), C.c_uint64(seed), _p(out))
    assert rc == 0
    return out


def gibbs_ex(eq, valid, eff_len, alphas_init, use_vbem, per_txp_prior, vb_prior, n_samples, thinning, no_gamma_draw,
             num_mapped_frags, seed, round0=0):
    """orc_gibbs_ex -> (samples [n_samples, M], mu and counts as the last round left them)."""
    lib = load()
    M = eq.n_txps
    out = np.zeros((n_samples, M))
    last_mu = np.zeros(M)
    last_cnt = np.zeros(M)
    rc = lib.orc_gibbs_ex(C.c_uint64(eq.n_classes), C.c_uint32(M), _p(eq.off), _p(eq.tids), _p(eq.weights),
                          _p(eq.counts), _p(np.ascontiguousarray(valid, dtype=np.uint8)),
                          _p(np.ascontiguousarray(eff_len, dtype=np.float64)),
                          _p(np.ascontiguousarray(alphas_init, dtype=np.float64)), C.c_int(use_vbem),
                          C.c_int(per_txp_prior), C.c_double(vb_prior), C.c_uint32(n_samples), C.c_uint32(thinning),
                          C.c_int(no_gamma_draw), C.c_double(num_mapped_frags), C.c_uint64(seed), C.c_uint32(round0),
                          _p(out), _p(last_mu), _p(last_cnt))
    assert rc == 0
    return out, last_mu, last_cnt


def gamma_draws(shape, scale, idx, rnd, seed):
    """orc_gamma_draw for every (shape, scale, i) triple: the sampler's gamma draws of round rnd."""
    lib = load()
    f = lib.orc_gamma_draw
    f.restype = C.c_double
    f.argtypes = [C.c_double, C.c_double, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    shape, scale, idx = np.broadcast_arrays(np.asarray(shape, dtype=np.float64), np.asarray(scale, dtype=np.float64),
                                            np.asarray(idx, dtype=np.uint64))
    return np.array([f(float(a), float(s), int(i), rnd, k0, k1) for a, s, i in zip(shape.ravel(), scale.ravel(),
                                                                                 idx.ravel())]).reshape(shape.shape)


# ---------------------------------------------------------------------------- Stage A
class orc_map_params(C.Structure):
    _fields_ = [
        ("k", C.c_uint32), ("stride", C.c_uint32), ("max_occs_per_hit", C.c_uint32), ("max_read_occ", C.c_uint32),
        ("max_frag_len", C.c_uint32), ("band", C.c_uint32), ("chain_gap", C.c_uint32), ("range_bins", C.c_uint32),
        ("ma", C.c_int32), ("mp", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32),
        ("hard_filter", C.c_int32), ("first_decoy", C.c_int32),
        ("consensus_frac", C.c_double), ("min_score_fraction", C.c_double), ("score_exp", C.c_double),
        ("min_aln_prob", C.c_double), ("decoy_threshold", C.c_double), ("fld_mean", C.c_double), ("fld_sd", C.c_double),
        ("num_pre_burnin", C.c_uint64), ("num_burnin", C.c_uint64),
        ("pre_merge_thresh", C.c_double), ("post_merge_thresh", C.c_double), ("orphan_thresh", C.c_double),
        ("allow_dovetail", C.c_int32), ("allow_orphans", C.c_int32), ("lib_type", C.c_int32), ("reserved3", C.c_int32),
    ]


class orc_map_counters(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("lookups", "postings", "seeds", "candidates", "kept", "label_entries", "mapped")]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


MAP_DEFAULTS = dict(k=31, stride=4, max_occs_per_hit=1000, max_read_occ=200, max_frag_len=1000, band=15, chain_gap=8,
                    range_bins=4, ma=2, mp=-4, go=6, ge=2, hard_filter=0, first_decoy=2**31 - 1, consensus_frac=0.65,
                    min_score_fraction=0.65, score_exp=1.0, min_aln_prob=1e-5, decoy_threshold=1.0, fld_mean=250.0,
                    fld_sd=25.0, num_pre_burnin=5000, num_burnin=5000000, pre_merge_thresh=0.75, post_merge_thresh=0.9,
                    orphan_thresh=0.95, allow_dovetail=0, allow_orphans=1, lib_type=0)


def map_params(**over):
    p = orc_map_params()
    d = dict(MAP_DEFAULTS); d.update(over)
    for k, v in d.items():
        setattr(p, k, v)
    return p


def pack_txome(txps):
    lens = np.array([t.shape[0] for t in txps], dtype=np.uint64)
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
    codes = np.ascontiguousarray(np.concatenate(txps).astype(np.uint8))
    return off, codes


class MapIndex:
    def __init__(self, txps, k=31):
        lib = load()
        lib.orc_index_build.restype = C.c_void_p
        lib.orc_index_n_kmers.restype = C.c_uint64
        lib.orc_index_n_kmers.argtypes = [C.c_void_p]
        self.off, self.codes = pack_txome(txps)
        self.n = len(txps)
        self.h = C.c_void_p(lib.orc_index_build(C.c_uint32(self.n), _p(self.off), _p(self.codes), C.c_uint32(k)))
        self.n_kmers = lib.orc_index_n_kmers(self.h)

    def __del__(self):
        try:
            load().orc_index_free.argtypes = [C.c_void_p]
            load().orc_index_free(self.h)
        except Exception:
            pass


def map_reads(index, p, left, right, frag_counter=0):
    lib = load()
    n, L = left.shape
    cap = p.max_read_occ
    left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
    out = dict(n_aln=np.zeros(n, dtype=np.uint32), tid=np.zeros((n, cap), dtype=np.uint32),
               score=np.zeros((n, cap), dtype=np.int32), prob=np.zeros((n, cap)), pos=np.zeros((n, cap), dtype=np.int32),
               mate_pos=np.zeros((n, cap), dtype=np.int32), flags=np.zeros((n, cap), dtype=np.uint8),
               flen=np.zeros((n, cap), dtype=np.int32), label=np.zeros((n, 2 * cap), dtype=np.uint32),
               weight=np.zeros((n, cap)))
    ctr = orc_map_counters()
    rc = lib.orc_map_reads(index.h, C.byref(p), _p(left), _p(right), C.c_uint32(n), C.c_uint32(L),
                           C.c_uint64(frag_counter), _p(out["n_aln"]), _p(out["tid"]), _p(out["score"]),
                           _p(out["prob"]), _p(out["pos"]), _p(out["mate_pos"]), _p(out["flags"]), _p(out["flen"]),
                           _p(out["label"]), _p(out["weight"]), C.byref(ctr))
    assert rc == 0
    out["counters"] = ctr.asdict()
    return out


def eq_aggregate(m, cap, binned=True):
    lib = load()
    lib.orc_eq_aggregate.restype = C.c_uint64
    n = m["n_aln"].shape[0]
    tot = int(m["n_aln"].sum())
    off = np.zeros(n + 1, dtype=np.uint64); ntx = np.zeros(n, dtype=np.uint32)
    lab = np.zeros(max(tot, 1), dtype=np.uint32); w = np.zeros(max(tot, 1)); cnt = np.zeros(n, dtype=np.uint64)
    nc = lib.orc_eq_aggregate(C.c_uint32(n), C.c_uint32(cap), C.c_int(1 if binned else 0), _p(m["n_aln"]),
                              _p(m["label"]), _p(m["weight"]), _p(off), _p(ntx), _p(lab), _p(w), _p(cnt))
    nc = int(nc)
    nn = int(off[nc])
    return dict(off=off[:nc + 1].copy(), ntx=ntx[:nc].copy(), tids=lab[:nn].copy(), weights=w[:nn].copy(), counts=cnt[:nc].copy())


class Online:
    """orc_online: the stateful oracle of the online phase (batched semantics, oracle/map_oracle.c)."""

    def __init__(self, index, p, seed=42, mini_batch=5000):
        lib = load()
        lib.orc_online_create.restype = C.c_void_p
        self.index, self.p = index, p
        self.h = C.c_void_p(lib.orc_online_create(index.h, C.byref(p), C.c_uint64(seed), C.c_uint32(mini_batch)))

    def batch(self, left, right):
        lib = load()
        n, L = left.shape
        cap = self.p.max_read_occ
        left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
        out = dict(n_aln=np.zeros(n, dtype=np.uint32), tid=np.zeros((n, cap), dtype=np.uint32),
                   score=np.zeros((n, cap), dtype=np.int32), prob=np.zeros((n, cap)), pos=np.zeros((n, cap), dtype=np.int32),
                   mate_pos=np.zeros((n, cap), dtype=np.int32), flags=np.zeros((n, cap), dtype=np.uint8),
                   flen=np.zeros((n, cap), dtype=np.int32), label=np.zeros((n, 2 * cap), dtype=np.uint32),
                   weight=np.zeros((n, cap)))
        ctr = orc_map_counters()
        rc = lib.orc_online_batch(self.h, _p(left), _p(right), C.c_uint32(n), C.c_uint32(L), _p(out["n_aln"]),
                                  _p(out["tid"]), _p(out["score"]), _p(out["prob"]), _p(out["pos"]), _p(out["mate_pos"]),
                                  _p(out["flags"]), _p(out["flen"]), _p(out["label"]), _p(out["weight"]), C.byref(ctr))
        assert rc == 0
        out["counters"] = ctr.asdict()
        return out

    def state(self):
        M, nf = self.index.n, self.p.max_frag_len + 1
        mass = np.zeros(M); hist = np.zeros(nf); le = np.zeros(M); sc = np.zeros(6, dtype=np.uint64)
        load().orc_online_state(self.h, _p(mass), _p(hist), _p(le), _p(sc))
        return dict(mass=mass, hist=hist, log_eff=le, assigned=int(sc[0]), frags_seen=int(sc[1]), timestep=int(sc[2]),
                    burned_in=int(sc[3]), min_val=int(sc[4]), tot=sc[5:6].view(np.float64)[0])

    def finish(self, off, tids, counts):
        M = self.index.n
        off = np.ascontiguousarray(off, dtype=np.uint64); tids = np.ascontiguousarray(tids, dtype=np.uint32)
        counts = np.ascontiguousarray(counts, dtype=np.uint64)
        proj = np.zeros(M); eff = np.zeros(M); uniq = np.zeros(M, dtype=np.uint64); tot = np.zeros(M, dtype=np.uint64)
        rc = load().orc_online_finish(self.h, C.c_uint64(len(counts)), _p(off), _p(tids), _p(counts), _p(proj), _p(eff),
                                      _p(uniq), _p(tot))
        assert rc == 0
        return dict(projected_counts=proj, eff_len=eff, unique_counts=uniq, total_counts=tot)

    def __del__(self):
        try:
            load().orc_online_free.argtypes = [C.c_void_p]
            load().orc_online_free(self.h)
        except Exception:
            pass


class orc_mate_info(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("lookups", "postings_all", "seeds", "cut_round", "distinct", "chains",
                                          "survivors", "straddle_seeds", "straddle_distinct")]

    def asdict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


ORC_CAND_DTYPE = np.dtype([("tid", np.uint32), ("ori", np.uint32), ("diag_c", np.int32), ("cov", np.uint32)])


def mate_candidates(index, p, read):
    """orc_mate_candidates: the candidates of one mate (structured array of ORC_CAND_DTYPE) and what its seeds look
    like (orc_mate_info as a dict)"""
    lib = load()
    read = np.ascontiguousarray(read, dtype=np.uint8)
    out = np.zeros(64, ORC_CAND_DTYPE)
    info = orc_mate_info()
    n = lib.orc_mate_candidates(index.h, C.byref(p), _p(read), C.c_uint32(read.shape[0]), _p(out), C.byref(info))
    return out[:n].copy(), info.asdict()
