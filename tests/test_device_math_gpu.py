"""The math primitives the parity claims rest on, run on the device (tests/dev_math_probe.cu) and checked against mpmath
at 50 digits and against their own host build:
  * sbm_det_exp / sbm_det_log (include/sb_detmath.h): Stage A's labels are bit-exact only because the device gives the
    host's bits.  Every binade of log's input, exp's subnormal results, its thresholds and range splits, NaN.
  * sb::fast_rcp (rcp.approx.ftz.f64 + two Newton steps on the device) and sb::exp_digamma_shifted (em_math.h), the VBEM
    transform, at its edges: x near DIGAMMA_MIN, the branch at x = 10, alpha up to 1e15, logNorm up to 35.
  * sb::digamma_pos (common.cuh), the EM's logNorm, on every branch of the Boost algorithm, and NaN for x <= 0.
  * sbmap::log_add and quant40 (map_core.h): device bits equal host bits.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "dev_math_probe.cu")
SO = os.path.join(ROOT, "tests", "_build", "libdevmathprobe.so")
HDRS = [os.path.join(ROOT, "include", "sb_detmath.h"), os.path.join(ROOT, "include", "salmon_b200.h")] + \
       [os.path.join(ROOT, "salmon_b200", "csrc", f) for f in ("em_math.h", "common.cuh", "map_core.h")]
NVCC = "/usr/local/cuda/bin/nvcc"
# the library's flags (Makefile: ARCH, NVCCFLAGS without the optional PTXAS_V); the device half keeps nvcc's default
# FMA contraction like the kernels, the host half is built without contraction like the oracle
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCCFLAGS = ["-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xcompiler", "-fopenmp"]
HOST_EXTRA = ["-Xcompiler", "-ffp-contract=off"]

OP_EXP, OP_LOG, OP_RCP, OP_EXP_DIGAMMA, OP_DIGAMMA, OP_LOG_ADD, OP_QUANT40 = range(7)
DIGAMMA_MIN = 1e-10
LN2 = 0.6931471805599453
EXP_HI = 7.09782712893383973096e+02      # sbm_det_exp: +inf above
EXP_LO = -7.45133219101941108420e+02     # sbm_det_exp: 0 below
TINY = 2.0 ** -28                        # sbm_det_exp: 1 + x below


def test_probe_flags_match_makefile():
    """the probe must see the contraction the library sees: its flags are the Makefile's"""
    mk = open(os.path.join(ROOT, "Makefile")).read()
    arch = re.search(r"^ARCH\s*:=\s*(.*)$", mk, re.M).group(1).split()
    flags = re.search(r"^NVCCFLAGS\s*:=\s*(.*)$", mk, re.M).group(1).replace("$(ARCH)", " ".join(arch))
    flags = flags.replace("$(PTXAS_V)", "").split()
    assert arch == ARCH
    assert flags == NVCCFLAGS
    assert "--fmad=false" not in flags and "-fmad=false" not in flags


def _lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if (not os.path.exists(SO)) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in [SRC] + HDRS):
        subprocess.check_call([NVCC, *NVCCFLAGS, *HOST_EXTRA, "-shared", "-o", SO + ".tmp", SRC])
        os.replace(SO + ".tmp", SO)
    lib = C.CDLL(SO)
    lib.dmp_run.restype = C.c_int
    lib.dmp_run.argtypes = [C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def probe():
    return _lib()


def run(probe, op, a, b=None, host=True):
    """(device, host) results as float64 arrays (int64 for quant40); host is None for a device-only op"""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.zeros_like(a) if b is None else np.ascontiguousarray(np.broadcast_to(b, a.shape), dtype=np.float64)
    dev = np.empty(a.shape, dtype=np.uint64)
    hst = np.empty(a.shape, dtype=np.uint64) if host else None
    rc = probe.dmp_run(op, len(a), a.ctypes.data, b.ctypes.data, dev.ctypes.data, hst.ctypes.data if host else None)
    assert rc == 0, rc
    dt = np.int64 if op == OP_QUANT40 else np.float64
    return dev.view(dt), (hst.view(dt) if host else None)


def mp():
    import mpmath
    mpmath.mp.dps = 50
    return mpmath


def ulp_err(got, want_mp):
    """|got - want| in units of the spacing of doubles at the correctly rounded want (denorm_min below the normals)"""
    m = mp()
    out = np.empty(len(got))
    for i, (g, w) in enumerate(zip(got, want_mp)):
        r = float(w)
        if np.isinf(r):
            out[i] = 0.0 if g == r else np.inf
            continue
        u = np.spacing(abs(r)) if r != 0.0 else 5e-324
        u = max(u, 5e-324)
        out[i] = float(abs(m.mpf(g) - w) / m.mpf(u))
    return out


def bits(x):
    return np.ascontiguousarray(x).view(np.uint64)


def assert_bits_equal(dev, host, args):
    bad = np.flatnonzero(bits(dev) != bits(host))
    assert len(bad) == 0, [(float(args[i]).hex(), float(dev[i]).hex(), float(host[i]).hex()) for i in bad[:8]]


def around(x, k=3):
    """x and its k neighbours on either side"""
    out = [x]
    lo = hi = x
    for _ in range(k):
        lo = np.nextafter(lo, -np.inf); hi = np.nextafter(hi, np.inf)
        out += [lo, hi]
    return out


# ---- sbm_det_exp ---------------------------------------------------------------------------------------------------
def exp_args():
    rng = np.random.default_rng(11)
    pts = [rng.uniform(-745.14, -708.3, 4000),                               # subnormal results
           rng.uniform(-708.3, 709.78, 4000), rng.uniform(-2.0, 2.0, 2000),
           np.concatenate([around(v, 4) for v in (EXP_HI, EXP_LO, -EXP_LO, -708.3964185322641)]),
           np.concatenate([around(s * v, 4) for s in (1, -1) for v in (0.5 * LN2, 1.5 * LN2, 0.34657359027997264,
                                                                         1.0397207708399179, TINY)]),
           rng.uniform(-TINY, TINY, 500), 10.0 ** rng.uniform(-320, np.log10(TINY), 500) * rng.choice([-1, 1], 500),
           np.array([0.0, -0.0, 5e-324, -5e-324, 1.0, -1.0, 700.0, -745.0, 1e-300])]
    return np.concatenate(pts)


@pytest.mark.gpu
def test_det_exp_device_equals_host_and_mpmath(probe):
    x = exp_args()
    dev, host = run(probe, OP_EXP, x)
    assert_bits_equal(dev, host, x)
    m = mp()
    fin = (x <= EXP_HI) & (x >= EXP_LO)
    err = ulp_err(dev[fin], [m.exp(m.mpf(v)) for v in x[fin]])
    assert err.max() <= 1.0, (float(err.max()), float(x[fin][np.argmax(err)]).hex())
    # the subnormal results are reached (k < -1021: the two-step scale)
    assert np.count_nonzero((dev > 0) & (dev < 2.2250738585072014e-308)) > 1000


@pytest.mark.gpu
def test_det_exp_documented_values(probe):
    over = np.array(around(EXP_HI, 4)[2::2] + [710.0, 1e300, np.inf])          # above 709.78: +inf
    under = np.array(around(EXP_LO, 4)[1::2] + [-746.0, -1e300, -np.inf])       # below -745.13: 0
    tiny = np.concatenate([around(TINY, 3)[1::2][1:], around(-TINY, 3)[2::2][1:],
                           np.random.default_rng(2).uniform(-TINY, TINY, 200), [0.0, -0.0, 5e-324, 1e-300]])
    tiny = tiny[np.abs(tiny) < TINY]
    assert len(tiny) > 200
    nan = np.array([0x7ff8000000000000, 0xfff8000000000000, 0x7ff8000000000123], dtype=np.uint64).view(np.float64)
    x = np.concatenate([over, under, tiny, nan])
    dev, host = run(probe, OP_EXP, x)
    assert_bits_equal(dev, host, x)
    n1, n2, n3 = len(over), len(over) + len(under), len(over) + len(under) + len(tiny)
    assert np.all(np.isposinf(dev[:n1]))
    assert np.all(bits(dev[n1:n2]) == 0)                                     # +0.0
    assert np.array_equal(bits(dev[n2:n3]), bits(1.0 + tiny))                # exactly 1 + x
    assert np.array_equal(bits(dev[n3:]), bits(nan))                         # the NaN itself, payload kept
    assert float(run(probe, OP_EXP, [EXP_HI])[0][0]) < np.inf                # the threshold itself is finite


# ---- sbm_det_log ---------------------------------------------------------------------------------------------------
def log_args():
    rng = np.random.default_rng(12)
    out = []
    # every normal binade: its first value, its last value and three random mantissas
    e = np.arange(1, 2047, dtype=np.uint64)
    for mant in (np.zeros(len(e), np.uint64), np.full(len(e), (1 << 52) - 1, np.uint64),
                 *[rng.integers(0, 1 << 52, len(e), dtype=np.uint64) for _ in range(3)]):
        out.append(((e << np.uint64(52)) | mant).view(np.float64))
    # every subnormal binade [2^j, 2^(j+1)) * denorm_min, j = 0..51
    for j in range(52):
        lo, hi = 1 << j, (1 << (j + 1)) - 1
        u = np.array([lo, hi] + list(rng.integers(lo, hi + 1, 3)), dtype=np.uint64)
        out.append(u.view(np.float64))
    # around 1, the sqrt(2) normalisation split (0x95f64) and 2^k, a dense spread
    out.append(np.concatenate([around(v, 4) for v in (1.0, 1.4142135623730951, 0.7071067811865476, 2.0, 0.5,
                                                        1.4142135623730951 * 2.0 ** 300, 1.4142135623730951 * 2.0 ** -1030)]))
    out.append(10.0 ** rng.uniform(-323, 308, 6000))
    out.append(rng.uniform(0.5, 2.0, 2000))
    return np.concatenate(out)


@pytest.mark.gpu
def test_det_log_device_equals_host_and_mpmath(probe):
    x = log_args()
    assert np.all(x > 0) and np.all(np.isfinite(x))
    assert np.count_nonzero(x < 2.2250738585072014e-308) >= 52 * 5
    dev, host = run(probe, OP_LOG, x)
    assert_bits_equal(dev, host, x)
    m = mp()
    err = ulp_err(dev, [m.log(m.mpf(v)) for v in x])
    assert err.max() <= 1.0, (float(err.max()), float(x[np.argmax(err)]).hex())
    assert bits(run(probe, OP_LOG, [1.0])[0])[0] == 0                         # log(1) = +0.0


@pytest.mark.gpu
def test_det_log_outside_its_domain_equals_host(probe):
    """callers guard x <= 0 and non-finite x; what comes out there is still the host's bits"""
    x = np.array([np.nan, np.inf, 0.0, -0.0, -1.0, -5e-324, -1e300])
    dev, host = run(probe, OP_LOG, x)
    assert_bits_equal(dev, host, x)


# ---- fast_rcp ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fast_rcp_within_1ulp(probe):
    rng = np.random.default_rng(13)
    # the operands exp_digamma_shifted hands it: x in [1e-10, 10) and x' Q(x) in [10 * 9!, 20 * 19!/10!), and x >= 10
    # up to the largest alphas; plus the whole normal range whose reciprocal is normal
    a = np.concatenate([10.0 ** rng.uniform(-10.5, 1.0, 4000), rng.uniform(3.6e6, 1.4e12, 2000),
                        10.0 ** rng.uniform(1.0, 16.0, 4000), 2.0 ** rng.uniform(-1022.0, 1021.99, 6000),
                        np.concatenate([around(2.0 ** k, 2) for k in (-1022, -1000, -1, 0, 1, 20, 52, 1000, 1021)]),
                        [DIGAMMA_MIN, DIGAMMA_MIN * (1 + 2.0 ** -40), 10.0, 1e12, 1e15]])
    a = a[(a >= 2.2250738585072014e-308) & (a < 2.0 ** 1022)]
    dev, host = run(probe, OP_RCP, a)
    assert np.array_equal(bits(host), bits(1.0 / a))                         # the host form is the division
    m = mp()
    err = ulp_err(dev, [1 / m.mpf(v) for v in a])
    assert err.max() <= 1.0, (float(err.max()), float(a[np.argmax(err)]).hex())


@pytest.mark.gpu
def test_fast_rcp_flushes_above_2_to_1022(probe):
    """Above 2^1022 the reciprocal is subnormal and rcp.approx.ftz flushes its seed to zero, which the Newton steps
    keep: fast_rcp(a) = +0 from 1.5 * 2^1022 up (measured on an H100).  Just above 2^1022 the seed still rounds to
    2^-1022 and the Newton steps reach the correctly rounded subnormal.  exp_digamma_shifted never gets there: its
    operands stay below 20 * 19!/10! and below the largest alphas (1e15 here)."""
    big = np.array([1.5 * 2.0 ** 1022, 2.0 ** 1023, 1.7976931348623157e308])
    dev, _ = run(probe, OP_RCP, big)
    assert np.all(bits(dev) == 0), [float(v).hex() for v in dev]
    a = np.array([2.0 ** 1022, np.nextafter(2.0 ** 1022, np.inf)])
    edge, _ = run(probe, OP_RCP, a)
    assert np.array_equal(bits(edge), bits(1.0 / a)), [float(v).hex() for v in edge]


# ---- exp_digamma_shifted -------------------------------------------------------------------------------------------
def edg_args():
    rng = np.random.default_rng(14)
    x = np.concatenate([
        np.array([DIGAMMA_MIN * (1 + 2.0 ** -40), DIGAMMA_MIN * 1.001, 1e-9, 1e-8, 1e-6, 1e-4, 0.01, 1.0, 2.0]),
        10.0 ** rng.uniform(-10.0, 15.0, 4000),
        np.concatenate([around(10.0, 40)]), 10.0 + rng.uniform(-1e-6, 1e-6, 400), rng.uniform(9.0, 11.0, 1500),
        rng.uniform(0.5, 12.0, 1500), 10.0 ** rng.uniform(11.0, 15.0, 500), [1e12, 1e15]])
    x = x[x > DIGAMMA_MIN]
    ln = np.concatenate([[0.0, 35.0], rng.uniform(0.0, 35.0, len(x) - 2)])
    return x, ln


@pytest.mark.gpu
def test_exp_digamma_shifted_device_vs_mpmath_and_host(probe):
    x, ln = edg_args()
    dev, host = run(probe, OP_EXP_DIGAMMA, x, ln)
    m = mp()
    psi = np.array([float(m.digamma(m.mpf(v))) for v in x])
    want = np.array([float(m.exp(m.digamma(m.mpf(v)) - m.mpf(l))) for v, l in zip(x, ln)])
    # test_em_math.py's tolerance: a few ulp of |psi - logNorm| in the exponent
    tol = 16 * np.spacing(np.maximum(1.0, np.maximum(np.abs(psi), np.abs(ln)))) + 4e-16
    ok = want > 1e-300
    assert np.count_nonzero(ok) > 0.7 * len(x)
    rel = np.abs(dev[ok] - want[ok]) / want[ok]
    assert np.all(rel <= tol[ok]), (float(rel.max()), float(x[ok][np.argmax(rel / tol[ok])]))
    assert np.all(dev[~ok] < 1e-299) and np.all(dev >= 0.0)
    # the device form (hardware reciprocal, contraction) against the host build: a few ulp of the exponent
    relh = np.abs(dev[ok] - host[ok]) / host[ok]
    assert np.all(relh <= tol[ok]), (float(relh.max()), float(x[ok][np.argmax(relh / tol[ok])]))
    # both sides of the branch at 10 are covered densely
    assert np.count_nonzero((x > 9.999) & (x < 10.0)) >= 100 and np.count_nonzero((x >= 10.0) & (x < 10.001)) >= 100


# ---- digamma_pos ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_digamma_pos_every_branch_vs_mpmath(probe):
    rng = np.random.default_rng(15)
    root = 1.4616321449683623
    x = np.concatenate([
        10.0 ** rng.uniform(-300, 0, 1500), rng.uniform(0.0, 1.0, 1000)[1:],   # x < 1: recurrence upwards
        np.concatenate([around(root, 20)]), root + rng.uniform(-0.05, 0.05, 1000),   # the root
        rng.uniform(1.0, 2.0, 1000), [1.0, 2.0, np.nextafter(2.0, 0), np.nextafter(1.0, 0)],   # [1, 2]
        rng.uniform(2.0, 10.0, 1500), around(10.0, 5),                          # (2, 10): recurrence downwards
        10.0 ** rng.uniform(1.0, 15.0, 1500), [1e12, 1e15, 1e300],              # >= 10: asymptotic
    ])
    x = x[x > 0]
    dev, _ = run(probe, OP_DIGAMMA, x, host=False)
    m = mp()
    want = [m.digamma(m.mpf(v)) for v in x]
    near = np.abs(x - root) < 0.05
    for i in range(len(x)):
        if near[i]:
            assert abs(m.mpf(dev[i]) - want[i]) < 4e-16, (float(x[i]).hex(), dev[i], want[i])
        else:
            assert abs((m.mpf(dev[i]) - want[i]) / want[i]) < 2e-15, (float(x[i]).hex(), dev[i], want[i])
    for lo, hi in ((0, 1), (1, 2), (2, 10), (10, np.inf)):
        assert np.count_nonzero((x >= lo) & (x < hi)) > 500


@pytest.mark.gpu
def test_digamma_pos_not_positive_is_nan(probe):
    """x <= 0 or NaN gives NaN at once instead of running the upward recurrence |x| times"""
    x = np.array([0.0, -0.0, -0.5, -3.5, -1000.0, np.nan])
    dev, _ = run(probe, OP_DIGAMMA, x, host=False)
    assert np.all(np.isnan(dev)), dev


# ---- log_add, quant40 ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_log_add_device_equals_host(probe):
    rng = np.random.default_rng(16)
    n = 20000
    x = np.concatenate([rng.uniform(-800, 50, n), rng.uniform(-5, 5, n)])
    y = np.concatenate([x[:n] + rng.normal(0, 30, n), x[n:] + rng.normal(0, 1e-6, n)])
    inf = np.inf
    special = [(inf, 3.0), (3.0, inf), (-inf, 3.0), (3.0, -inf), (inf, inf), (-inf, -inf), (inf, -inf), (-inf, inf),
               (inf, -0.5), (-700.0, inf), (2.0, 2.0), (-1.0, -1.0), (0.0, -0.0), (-745.5, 0.0), (0.0, -745.5),
               (710.0, -30.0), (-1e300, 1.0)]
    x = np.concatenate([x, [s[0] for s in special]])
    y = np.concatenate([y, [s[1] for s in special]])
    dev, host = run(probe, OP_LOG_ADD, x, y)
    assert_bits_equal(dev, host, x)
    # the LOG_0 (= +inf) rules: an infinite operand of either sign returns the other operand
    k = len(x) - len(special)
    assert dev[k + 0] == 3.0 and dev[k + 1] == 3.0 and dev[k + 2] == 3.0 and dev[k + 3] == 3.0
    assert dev[k + 4] == inf and dev[k + 5] == -inf and dev[k + 6] == -inf and dev[k + 7] == inf
    assert dev[k + 8] == -0.5 and dev[k + 9] == -700.0


@pytest.mark.gpu
def test_quant40_ties_device_equals_host(probe):
    """exact ties (k + 1/2) 2^-40 round to even on both sides"""
    k = np.concatenate([np.arange(-20, 21), np.array([1 << 20, (1 << 20) + 1, 12345678901, (1 << 51) - 1]),
                        np.random.default_rng(17).integers(-(1 << 50), 1 << 50, 2000)])
    x = np.concatenate([(k + 0.5) * 2.0 ** -40, k * 2.0 ** -40, (k + 0.25) * 2.0 ** -40])
    assert np.array_equal(x * 2.0 ** 40, np.concatenate([k + 0.5, k, k + 0.25]))   # the products are exact
    dev, host = run(probe, OP_QUANT40, x)
    assert np.array_equal(dev, host)
    want = np.array([round(float(v)) for v in x * 2.0 ** 40], dtype=np.int64)   # Python rounds half to even
    assert np.array_equal(dev, want)
