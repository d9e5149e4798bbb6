"""Every library object gives back all the CUDA resources it made, and the hot calls reuse their buffers: read through
sb_debug_device_memory (live buffers / streams / events, live bytes, allocations made), which sees the library alone
-- the device's free memory is noise on a shared GPU."""
import gc
import os
import threading

import numpy as np
import pytest

from salmon_b200 import EMContext, default_params
from salmon_b200 import _capi
from salmon_b200._capi import EqBuilder, Index, MapContext, SamSink, map_default_params
from salmon_b200.synth import synth_eq, synth_reads, synth_txome

pytestmark = pytest.mark.gpu


def mem():
    gc.collect()   # objects of earlier tests that are only waiting for the collector release theirs now
    out = np.zeros(3, dtype=np.uint64)
    assert _capi.load().sb_debug_device_memory(out.ctypes.data) == 0
    return [int(x) for x in out]


def live(m):
    return m[:2]


@pytest.fixture(scope="module")
def em_inputs():
    return synth_eq(seed=9, C=30000, M=8000, total_count=600000)


def test_em_context_life(em_inputs):
    eq, proj, eff, uniq = em_inputs
    nmapped = float(eq.counts.sum())
    base = mem()
    for _ in range(3):
        c = EMContext(0)
        alpha, st, ok = c.optimize(eq, default_params(), proj, eff, uniq)
        assert ok
        c.bootstrap(default_params(min_iter=20, max_iter=50), nmapped, 2, 11)
        c.gibbs(alpha, 1, 1, 1e-2, n_samples=3, thinning=2, no_gamma_draw=0, num_mapped_frags=nmapped, seed=5)
        c.close()
        assert live(mem()) == live(base)
    for _ in range(2):
        c = EMContext(0)
        c.peer_loopback(eq.n_txps)
        c.optimize(eq, default_params(min_iter=5, max_iter=5), proj, eff, uniq)
        c.close()
        assert live(mem()) == live(base)
    assert mem()[2] > base[2]


def test_em_repeated_calls_allocate_nothing(em_inputs):
    eq, proj, eff, uniq = em_inputs
    nmapped = float(eq.counts.sum())
    p = default_params(min_iter=30, max_iter=30)
    c = EMContext(0)
    try:
        alpha, _, _ = c.optimize(eq, p, proj, eff, uniq)
        made = mem()[2]
        c.optimize(eq, p, proj, eff, uniq)
        assert mem()[2] == made
        t = threading.Thread(target=lambda: c.optimize(eq, p, proj, eff, uniq))   # the owner is the context's
        t.start(); t.join()
        assert mem()[2] == made
        c.upload(eq, proj, eff, uniq); c.prepare(p); c.run()
        assert mem()[2] == made
        pb = default_params(min_iter=20, max_iter=50)
        c.bootstrap(pb, nmapped, 1, 3)
        c.gibbs(alpha, 1, 1, 1e-2, n_samples=1, thinning=2, no_gamma_draw=0, num_mapped_frags=nmapped, seed=5)
        made = mem()[2]
        c.bootstrap(pb, nmapped, 4, 4)    # rounds after the first
        c.gibbs(alpha, 1, 1, 1e-2, n_samples=4, thinning=2, no_gamma_draw=0, num_mapped_frags=nmapped, seed=6)
        assert mem()[2] == made
    finally:
        c.close()


def test_map_context_and_index_life(tmp_path):
    txps, _ = synth_txome(seed=3, n_genes=60)
    left, right, _ = synth_reads(txps, seed=5, n=1500)
    names = [f"r{i}" for i in range(len(left))]
    base = mem()
    for _ in range(2):
        ix = Index(txps)
        for paired in (True, False):
            mp = map_default_params(recover_orphans=1, softclip=2) if paired else map_default_params(lib_type=3, softclip=2)
            r = right if paired else None
            mc = MapContext(ix, mp, batch_cap=2048, max_read_len=100)
            sink = SamSink(ix, os.devnull, str(tmp_path / "un.txt"))
            mc.attach_sam(sink)
            mc.map_batch_sam(left, r, names)
            mc.attach_sam(None)
            sink.close()
            mc.map_batch(left, r)
            mc.reset()
            made = mem()[2]
            mc.map_batch(left, r)      # the buffers and the arena are large enough already
            assert mem()[2] == made
            res = mc.finish()
            assert len(res["counts"]) > 0
            mc.close()
        ix.close()
        assert live(mem()) == live(base)


def test_eq_builder_life(em_inputs):
    eq = em_inputs[0]
    base = mem()
    for _ in range(3):
        b = EqBuilder(eq.n_txps)
        b.from_host(eq)
        b.from_host(eq)
        t = b.finish()
        assert len(t["counts"]) > 0
        b.close()
        assert live(mem()) == live(base)
