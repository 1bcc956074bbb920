"""The P-256 squaring, the Jacobian + affine mixed addition and the Jacobian fixed-base walk, against exact integers and
oracle/curves.py.

Field<FpP256>::sqr is a multiplier of its own on the device (p256_sqr_body, 36 products); the fixed-base walks
(p256_accum_fixed / p256_accum_fixed_jac) accumulate with jac_madd, which is not complete, so each of its exceptional
inputs (the identity accumulator, P + P, P + (-P)) is driven here on purpose, on its own and inside whole table walks
whose partial sums are crafted to meet the next entry or its negative.  The probe is tests/probe/zk_probe_jac.cu
(zk_probe.cu plus these operations).  Every check runs on its host build; with -m gpu the same checks run on the
sm_90a build.
"""
import os
import random
import time

import numpy as np
import pytest

from oracle.curves import p256
from test_arith_edges import FIELDS, NAMES, OP_MUL, W, Probe, catalogue, ints, limbs, mont_ref, p256_affine, quotient_pairs

P, N, R = p256.p, p256.order, 1 << 256
RINV = pow(R, -1, P)


@pytest.fixture(scope='module')
def probe_host():
    import __graft_entry__ as g
    g.build_probe(host=True, jac=True)
    return Probe(g.PROBE_JAC_HOST)


@pytest.fixture(scope='module')
def probe_dev():
    import __graft_entry__ as g
    g.build_probe(jac=True)
    return Probe(g.PROBE_JAC)


def sqr_call(Pr, field, vals):
    import ctypes as C
    L = Pr.lib
    L.probe_sqr.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.probe_sqr.restype = C.c_int
    a = limbs(vals)
    out = np.zeros_like(a)
    assert L.probe_sqr(field, len(a), a.ctypes.data, out.ctypes.data) == 0
    return ints(out)


def jac_madd_call(Pr, rows):
    """rows: [(X, Y, Z, x, y)] Montgomery -> [(X3, Y3, Z3)]"""
    import ctypes as C
    L = Pr.lib
    L.probe_jac_madd.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    L.probe_jac_madd.restype = C.c_int
    inp = limbs([c for r in rows for c in r], 8).reshape(len(rows), 40)
    out = np.zeros((len(rows), 24), np.uint32)
    assert L.probe_jac_madd(len(rows), inp.ctypes.data, out.ctypes.data) == 0
    return [ints(o.reshape(3, 8)) for o in out]


def mont(v):
    return v % P * R % P


# ------------------------------------------------------------------------------------------------ squaring
def check_sqr(Pr, field):
    p, n, lazy = FIELDS[field]
    cat = catalogue(field) + [a for a, _ in quotient_pairs(field)]
    want = []
    for a in cat:
        t = mont_ref(a, a, p, n)
        want.append(t if lazy else (t - p if t >= p else t))
    got = sqr_call(Pr, field, cat)
    for a, g, w in zip(cat, got, want):
        assert g == w, (NAMES[field], hex(a), hex(g), hex(w))
    return cat, got


@pytest.mark.parametrize('field', [0, 1, 2, 3], ids=lambda f: NAMES[f])
def test_sqr_edges_host(probe_host, field):
    check_sqr(probe_host, field)


@pytest.mark.gpu
@pytest.mark.parametrize('field', [0, 1, 2, 3], ids=lambda f: NAMES[f])
def test_sqr_edges_device(probe_dev, field):
    cat, got = check_sqr(probe_dev, field)
    assert got == probe_dev.field(field, OP_MUL, cat, cat), NAMES[field]   # the squaring is mul(a, a)


# squarings compared by the device differential (ZKA_PROBE_DIFF_PRODUCTS overrides), as in test_arith_edges
DIFF_SQUARES = int(os.environ.get('ZKA_PROBE_DIFF_PRODUCTS', str(1 << 30)))


@pytest.mark.gpu
def test_sqr_differential_device(probe_dev, capsys):
    """~10^9 hashed p256.p operands (random lengths, all-ones / zero limbs, just below p): p256_sqr_body against the
    generic CIOS mul_generic(a, a), plus the output bound.  Mismatches are re-derived in Python."""
    import ctypes as C
    L = probe_dev.lib
    L.probe_sqr_diff.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.probe_sqr_diff.restype = C.c_int
    m = np.zeros(1, np.uint32)
    bad = np.zeros((16, 2, W), np.uint32)
    t0 = time.perf_counter()
    assert L.probe_sqr_diff(0, 0x5ec0, DIFF_SQUARES, 0, 64, m.ctypes.data, bad.ctypes.data) == 0
    dt = time.perf_counter() - t0
    mism = int(m[0])
    with capsys.disabled():
        print(f'\n[probe] p256.p: {DIFF_SQUARES} squarings, {mism} mismatches, {dt:.2f} s')
    for a, r in (ints(x) for x in bad[:min(mism, 16)]):
        want = mont_ref(a, a, P, 8)
        want = want - P if want >= P else want
        assert r != want or r >= P, 'device mismatch not confirmed in Python'
    assert mism == 0, [hex(a) for a, _ in (ints(x) for x in bad[:min(mism, 16)])]


# ------------------------------------------------------------------------------------------------ jac_madd
def jac_of(pt, rnd):
    """(x z^2, y z^3, z) with a random z; the identity as (1 : 1 : 0) or (t^2 : t^3 : 0)"""
    a = p256_affine(pt)
    if a is None:
        t = rnd.choice([1, rnd.randrange(1, P)])
        return (mont(t * t), mont(t * t * t), 0, 0)
    z = rnd.randrange(1, P)
    return (mont(a[0] * z * z), mont(a[1] * z ** 3), 0, mont(z))


def from_jac(X, Y, Z):
    """Montgomery Jacobian -> None (identity) or canonical affine (x, y)"""
    X, Y, Z = X * RINV % P, Y * RINV % P, Z * RINV % P
    if Z == 0:
        assert Y != 0, 'Jacobian identity with Y = 0'
        return None
    zi = pow(Z, -1, P)
    return X * zi * zi % P, Y * zi ** 3 % P


def from_hom(X, Y, Z):
    X, Y, Z = X * RINV % P, Y * RINV % P, Z * RINV % P
    if Z == 0:
        assert Y != 0 and X == 0, 'homogeneous identity must be (0 : Y : 0)'
        return None
    zi = pow(Z, -1, P)
    return X * zi % P, Y * zi % P


def check_jac_madd(Pr):
    rnd = random.Random(11)
    G = p256.generator()
    pts = [G, G.neg(), G.dbl(), G.mul(p256.new_scalar(N - 2))]
    pts += [G.mul(p256.new_scalar(rnd.randrange(1, N))) for _ in range(6)]
    cases = []
    for q in pts:
        cases.append((p256.identity(), q))        # identity accumulator
        cases.append((q, q))                      # H = 0, r = 0: doubling
        cases.append((q.neg(), q))                # H = 0, r != 0: the identity
        for p in pts:
            cases.append((p, q))                  # generic (and the collisions among pts)
    rows = []
    for p, q in cases:
        qa = p256_affine(q)
        X, Y, _, Z = jac_of(p, rnd)
        rows.append((X, Y, Z, mont(qa[0]), mont(qa[1])))
    outs = jac_madd_call(Pr, rows)
    for (p, q), o in zip(cases, outs):
        assert from_jac(*o) == p256_affine(p.add(q)), ('jac_madd', p256_affine(p), p256_affine(q))
    kinds = {'identity + P': 0, 'P + P': 0, 'P + (-P)': 0}
    for p, q in cases:
        if p256_affine(p) is None:
            kinds['identity + P'] += 1
        elif p256_affine(p) == p256_affine(q):
            kinds['P + P'] += 1
        elif p256_affine(p.add(q)) is None:
            kinds['P + (-P)'] += 1
    assert all(v >= len(pts) for v in kinds.values()), kinds


def test_jac_madd_host(probe_host):
    check_jac_madd(probe_host)


@pytest.mark.gpu
def test_jac_madd_device(probe_dev):
    check_jac_madd(probe_dev)


# ------------------------------------------------------------------------------------------------ fixed-base walks
def fb_windows(w):
    return (256 + w) // w


def fb_entries(w):
    return (1 << (w - 1)) + 1


def signed_digits(k, w):
    """zk_ops.cuh signed_digit: k = sum_j d_j 2^(w j), d_j in [-2^(w-1), 2^(w-1)]"""
    out, carry, half = [], 0, 1 << (w - 1)
    for j in range(fb_windows(w)):
        d = carry + ((k >> (j * w)) & ((1 << w) - 1))
        carry = 1 if d > half else 0
        out.append(d - (1 << w) if d > half else d)
    assert sum(d << (w * j) for j, d in enumerate(out)) == k
    return out


_TABLES = {}


def table(w, base_k):
    """[fb_windows(w)][fb_entries(w)][16] affine Montgomery entries d 2^(w j) B (entry 0: B itself, never read)"""
    key = (w, base_k)
    if key not in _TABLES:
        B = p256.generator().mul(p256.new_scalar(base_k))
        tab = np.zeros((fb_windows(w), fb_entries(w), 16), np.uint32)
        pw = B
        ba = p256_affine(B)
        for j in range(fb_windows(w)):
            acc = pw
            tab[j, 0] = limbs([mont(ba[0]), mont(ba[1])], 8).reshape(16)
            for d in range(1, fb_entries(w)):
                a = p256_affine(acc)
                tab[j, d] = limbs([mont(a[0]), mont(a[1])], 8).reshape(16)
                acc = acc.add(pw)
            for _ in range(w):
                pw = pw.dbl()
        _TABLES[key] = (B, tab)
    return _TABLES[key]


def accum_call(Pr, jac, w, tab, scalars, accs):
    import ctypes as C
    L = Pr.lib
    L.probe_p256_accum.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4
    L.probe_p256_accum.restype = C.c_int
    s = limbs(scalars, 8)
    a = limbs([c for acc in accs for c in acc], 8).reshape(len(accs), 24)
    out = np.zeros_like(a)
    assert L.probe_p256_accum(jac, w, len(s), tab.ctypes.data, s.ctypes.data, a.ctypes.data, out.ctypes.data) == 0
    return [ints(o.reshape(3, 8)) for o in out]


def walk_cases(w, rnd):
    """(k, s): the walk adds s B on top of k B.  k is crafted so that the partial sum before window j equals the entry
    added there (doubling) or its negative (identity), which is what a key that is a small multiple of G does."""
    cases = []
    for s in (0, 1, N - 1, 2, 1 << (w * 3), (1 << 255), (1 << w) - 1, N - (1 << w)):   # small, top-only, zero windows
        for k in (0, 1, 5, N - 1):
            cases.append((k, s))
    for _ in range(6):
        s = rnd.randrange(N)
        d = signed_digits(s, w)
        for j in [0, 1, 2] + rnd.sample(range(3, fb_windows(w) - 1), 3):
            if d[j] == 0:
                continue
            before = sum(di << (w * i) for i, di in enumerate(d[:j]))
            step = d[j] << (w * j)
            cases.append(((step - before) % N, s))         # partial sum == next entry: P + P
            cases.append(((-step - before) % N, s))        # partial sum == -(next entry): P + (-P)
        cases.append((rnd.randrange(N), s))
    return cases


def check_walk(Pr, w, jac):
    rnd = random.Random(100 * w + jac)
    B, tab = table(w, 0x5eed1234abcd)
    cases = walk_cases(w, rnd)
    accs = []
    for k, _ in cases:
        pt = B.mul(p256.new_scalar(k)) if k else p256.identity()
        a = p256_affine(pt)
        if jac:
            X, Y, _, Z = jac_of(pt, rnd)
            accs.append((X, Y, Z))
        else:
            z = rnd.randrange(1, P)
            accs.append((0, mont(z), 0) if a is None else (mont(a[0] * z), mont(a[1] * z), mont(z)))
    outs = accum_call(Pr, jac, w, tab, [s for _, s in cases], accs)
    conv = from_jac if jac else from_hom
    for (k, s), o in zip(cases, outs):
        want = p256_affine(B.mul(p256.new_scalar((k + s) % N))) if (k + s) % N else None
        assert conv(*o) == want, ('accum_fixed' + ('_jac' if jac else ''), w, hex(k), hex(s))


@pytest.mark.parametrize('jac', [1, 0], ids=['jacobian', 'homogeneous'])
@pytest.mark.parametrize('w', [5, 8])
def test_accum_fixed_host(probe_host, w, jac):
    check_walk(probe_host, w, jac)


@pytest.mark.gpu
@pytest.mark.parametrize('jac', [1, 0], ids=['jacobian', 'homogeneous'])
@pytest.mark.parametrize('w', [5, 8])
def test_accum_fixed_device(probe_dev, w, jac):
    check_walk(probe_dev, w, jac)
