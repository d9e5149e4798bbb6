"""EM kernel sweep on BASELINE config 2 (dev helper): every setting is checked against the first one.
usage: sweep_em.py iters "key=value:key=value,key=value:..." [vbem]      (settings separated by commas)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from salmon_b200 import EMContext, default_params
from salmon_b200.synth import synth_eq

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 300
settings = [dict((kv.split("=")[0], int(kv.split("=")[1])) for kv in x.split(":") if kv) for x in sys.argv[2].split(",")]
vbem = int(sys.argv[3]) if len(sys.argv) > 3 else 1
eq, proj, eff, uniq = synth_eq(seed=1)
ctx = EMContext(0)
p = default_params(min_iter=iters, max_iter=iters, use_vbem=vbem)
ctx.upload(eq, proj, eff, uniq)
ref = None
for stg in settings:
    for k, v in stg.items():
        ctx.set_option(k, v)
    try:
        st = ctx.prepare(p)
        best = 1e30
        for rep in range(3):
            ctx.flush_l2()
            r = ctx.run()
            best = min(best, r.loop_kernel_ms)
        a, s, ok = ctx.download()
    except Exception as e:  # noqa
        print(stg, "FAILED", e, flush=True)
        continue
    if ref is None:
        ref = a
    sb = ctx.info("stream_bytes")
    print(f"{str(stg):70s} prepare {st.prepare_ms:6.2f} ms  loop {best / iters * 1e3:7.2f} us/iter  {iters / (best / 1e3):8.0f} iters/s  "
          f"stream {sb / 1e6:6.2f} MB/iter = {sb * iters / (best / 1e3) / 1e9:6.0f} GB/s  "
          f"fallback rows {ctx.info('fallback_rows_cm')}/{ctx.info('fallback_rows_tm')}  "
          f"maxdiff vs first {np.max(np.abs(a - ref) / np.maximum(ref, 1e-6)):.1e}", flush=True)
