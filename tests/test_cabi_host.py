"""CPU tests (-m "not gpu") of the product's C-ABI library: it loads, exports every symbol
include/rbf_b200.h declares, its exact host-side scalars match the golden vectors, and it
refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.util import golden_json

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


@pytest.fixture(scope="module")
def cabi():
    from new_bloom_filter_repo_b200 import build, _cabi
    build.build()
    return _cabi


def test_header_symbols_exported(cabi):
    hdr = open(os.path.join(ROOT, "include", "rbf_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(rbf_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 45
    L = C.CDLL(cabi.SO_PATH)
    missing = [n for n in declared if not hasattr(L, n)]
    assert not missing, missing
    assert sorted(cabi.EXPORTS) == declared
    assert cabi.lib().rbf_abi_version() == 4


def test_host_xxh64_matches_golden(cabi):
    g = golden_json("xxh64_kat.json")
    L = cabi.lib()
    for rec in g["decimal"]:
        for s, d in zip(g["seeds"], rec["digests"]):
            assert format(L.rbf_hash_decimal(rec["item"], s), "016x") == d
            assert format(L.rbf_hash_decimal_century(rec["item"], s), "016x") == d      # the route the kernels take
    for rec in g["strings"]:
        b = rec["s"].encode("utf-8")
        for s, d in zip(g["seeds"], rec["digests"]):
            assert format(cabi.xxh64(b, s), "016x") == d


def test_century_route_dense_ranges(cabi):
    L = cabi.lib()
    rng = np.random.default_rng(3)
    items = np.concatenate([np.arange(0, 12000), np.arange(99000, 101200), np.arange(999900, 1000200),
                            np.arange(9999900, 10000200), np.arange(99999900, 100000200),
                            np.arange(999999900, 1000000200), np.arange(2 ** 32 - 300, 2 ** 32),
                            rng.integers(0, 2 ** 32, 20000)])
    for seed in (0x12345678, 0x87654321, 999):
        for it in items[::3]:
            it = int(it)
            assert L.rbf_hash_decimal(it, seed) == L.rbf_hash_decimal_century(it, seed), it


def test_probe_index_and_threshold(cabi):
    g = golden_json("filter_kat.json")
    L = cabi.lib()
    for rec in g["filters"]:
        T = cabi.activation_threshold(float.fromhex(rec["p_activation"]))
        for it, probes, act in zip(rec["items"], rec["probes"], rec["activation"]):
            b = str(it).encode()
            h1, h2 = cabi.xxh64(b, 0x12345678), cabi.xxh64(b, 0x87654321)
            assert [L.rbf_probe_index(h1, h2, i, rec["size"]) for i in range(rec["floor_k"] + 1)] == probes
            assert (cabi.xxh64(b, 999) < T) == act
    a = golden_json("activation_kat.json")
    for rec in a["thresholds"]:
        T = int(rec["T"], 16)
        if T < 2 ** 64:
            assert cabi.activation_threshold(float.fromhex(rec["p"])) == T


def test_optimal_params_matches_reference(cabi):
    g = golden_json("params_kat.json")
    for rec in g["cases"]:
        coded, p, k, l = cabi.optimal_params(rec["n"], rec["ones"])
        assert float(p).hex() == rec["p"]
        kr, lr = float.fromhex(rec["k"]), rec["l"]
        ref_coded = not (float.fromhex(rec["p"]) >= 0.32453) and not (lr == 0 or lr >= rec["n"])
        assert coded == ref_coded, rec
        if coded:
            assert (float(k).hex(), l) == (float(kr).hex(), lr), rec


def test_no_cpu_fallback(cabi):
    """Without a GPU the product must raise, not compute (run only where no GPU is visible)."""
    h = C.c_void_p()
    rc = cabi.lib().rbf_ctx_create(0, C.byref(h))
    if rc == 0:
        cabi.lib().rbf_ctx_destroy(h)
        pytest.skip("a GPU is present")
    assert rc == -3
    assert b"no CPU fallback" in cabi.lib().rbf_last_global_error()
    import new_bloom_filter_repo_b200 as pkg
    with pytest.raises(pkg.RbfError):
        pkg.BloomFilterCompressor().compress(np.zeros(100, dtype=np.uint8))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "new_bloom_filter_repo_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.replace("no oracle", ""), f


# ------------------------------------------------------------------ randomized differentials of the exact host scalars
def test_probe_index_random_vs_bigint(cabi):
    """(h1 + i*h2) % m in unbounded integers (ivc:79-81) for random 64-bit hashes and awkward moduli."""
    L = cabi.lib()
    rng = np.random.default_rng(11)
    ms = [1, 2, 3, 997, 2 ** 16, 2 ** 23, 2 ** 23 + 1, 1908859, 2 ** 30 - 1, 2 ** 30, 2 ** 30 + 1, 2 ** 31, 2 ** 32 - 1]
    ms += [int(x) for x in rng.integers(1, 2 ** 32, 300)]
    for m in ms:
        for _ in range(20):
            h1, h2 = (int(x) for x in rng.integers(0, 2 ** 64, 2, dtype=np.uint64))
            if rng.random() < 0.1:
                h1, h2 = 2 ** 64 - 1, 2 ** 64 - 1 - int(rng.integers(0, 3))
            for i in (0, 1, 2, 7, 63):
                assert L.rbf_probe_index(h1, h2, i, m) == (h1 + i * h2) % m, (h1, h2, i, m)


def test_activation_threshold_is_the_exact_cut(cabi):
    """h < T  <=>  h / (2**64 - 1) < p with Python's correctly rounded int/int division (ivc:95-97)."""
    rng = np.random.default_rng(12)
    D = 2 ** 64 - 1
    ps = [0.5, 0.25, 0.1, 0.2999999999999998, 1e-9, 1 - 2 ** -53, 2 ** -64, 2 ** -60, 0.9999999999]
    ps += [float(x) for x in rng.random(400)] + [float(x) for x in rng.random(100) * 1e-6]
    for p in ps:
        T = cabi.activation_threshold(p)
        assert 0 <= T <= 2 ** 64
        if T > 0:
            assert (T - 1) / D < p, (p, T)
        if T < 2 ** 64:
            assert not (T / D < p), (p, T)
    assert cabi.activation_threshold(0.0) == 0


def test_optimal_params_random_vs_reference_expression(cabi):
    """_calculate_optimal_params (ivc:161-196) restated with Python floats, against the library's host routine."""
    import math
    P_STAR = 0.32453

    def ref(n, ones):
        p = ones / n
        if p >= P_STAR:
            return False, p, 0.0, 0
        if p <= 0.0001 or p >= P_STAR:
            return False, p, 0.0, 0
        L = math.log(2.0)
        k = math.log2((1.0 - p) * math.pow(L, 2.0) / p)
        if k <= 0 or math.isnan(k):
            return False, p, 0.0, 0
        l = int(p * n * k * (1.0 / L))
        k, l = max(0.1, k), max(1, l)
        return not (l == 0 or l >= n), p, k, l

    rng = np.random.default_rng(13)
    cases = [(n, int(n * f)) for n in (4096, 2073600, 8294400, 33177600) for f in (0.0, 0.00009, 0.0001, 0.00011, 0.05, 0.3245, 0.32453, 0.3246, 0.5, 1.0)]
    for _ in range(3000):
        n = int(rng.integers(1, 40_000_000))
        cases.append((n, int(rng.integers(0, n + 1) * (rng.random() ** 3))))
    for n, ones in cases:
        coded, p, k, l = cabi.optimal_params(n, ones)
        rc, rp, rk, rl = ref(n, ones)
        assert float(p).hex() == float(rp).hex(), (n, ones)
        assert bool(coded) == rc, (n, ones, k, l, rk, rl)
        if rc:
            assert (float(k).hex(), l) == (float(rk).hex(), rl), (n, ones)


def test_ctx_as_first_call_does_not_deadlock():
    """`ImprovedVideoCompressor()` as the very first use of the package calls _cabi.ctx() before _cabi.lib(): the library load
    happens under the context lock, which therefore has to be re-entrant (a plain Lock hung scripts/gop_fps.py for good).
    Run in a fresh interpreter with a watchdog; without a GPU the call must fail with RbfError, not hang."""
    import subprocess
    import sys
    code = ("import faulthandler, sys; faulthandler.dump_traceback_later(60, exit=True)\n"
            "sys.path.insert(0, %r)\n"
            "from new_bloom_filter_repo_b200 import _cabi\n"
            "try:\n"
            "    _cabi.ctx()\n"
            "    print('ctx ok')\n"
            "except _cabi.RbfError as e:\n"
            "    print('RbfError', str(e)[:60])\n") % ROOT
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr[-500:]
    assert "ctx ok" in res.stdout or "RbfError" in res.stdout
