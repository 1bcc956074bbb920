"""Field operations and scalar recoders at the edges of their documented domains, against exact integer references.

The probe (tests/probe/zk_probe.cu) runs the library's own Field<F> operations and digit recoders on raw 32-bit limbs:
no Montgomery conversion, reduction or byte encoding on the way in, so operands can sit anywhere in the domain each
operation documents (tom.p: lazy values below 2^13 p; the strict fields: canonical).  The host build runs in the CPU
suite; the sm_90a build (the PTX multipliers) runs under -m gpu and must agree with Python and with the host build.
"""
import os
import random
import time

import numpy as np
import pytest

from oracle.curves import p256, tomEdwards256 as tom, war256

W = 9            # words per element in the probe's buffers
DIGIT_ROW = 132

# field index -> (modulus, limbs, lazy)
FIELDS = {0: (p256.p, 8, False), 1: (p256.order, 8, False), 2: (tom.p, 9, True), 3: (war256.p, 8, False)}
NAMES = {0: 'p256.p', 1: 'p256.n', 2: 'tom.p', 3: 'war.p'}
(OP_MUL, OP_MUL_GENERIC, OP_MUL_INL, OP_ADD, OP_SUB, OP_NEG, OP_REDUCE, OP_FROM_MONT, OP_IS_ZERO, OP_EQ,
 OP_INV) = range(11)
K_SIGNED, K_MSM6, K_MSM4, K_AGG = range(4)
LAZY_BITS = 13   # tom.p operands of mul / from_mont / inv are below 2^13 p (zk_field_ptx.cuh, DESIGN 4)


class Probe:
    def __init__(self, path):
        import ctypes as C
        self.lib = L = C.CDLL(path)
        P = C.c_void_p
        L.probe_field.argtypes = [C.c_int, C.c_int, C.c_int, P, P, P]
        L.probe_mul_diff.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.c_int, P, P]
        L.probe_digits.argtypes = [C.c_int, C.c_int, C.c_int, P, P, P]
        for f in (L.probe_field, L.probe_mul_diff, L.probe_digits):
            f.restype = C.c_int

    def field(self, field, op, a, b=None):
        a = limbs(a)
        b = limbs(b) if b is not None else np.zeros_like(a)
        out = np.zeros_like(a)
        assert self.lib.probe_field(field, op, len(a), a.ctypes.data, b.ctypes.data, out.ctypes.data) == 0
        return ints(out)

    def mul_diff(self, field, seed, count, bound_bits, per=64):
        m = np.zeros(1, np.uint32)
        bad = np.zeros((16, 3, W), np.uint32)
        assert self.lib.probe_mul_diff(field, seed, count, bound_bits, per, m.ctypes.data, bad.ctypes.data) == 0
        return int(m[0]), bad

    def digits(self, kind, w, scalars):
        s = limbs(scalars, 8)
        rows = 2 if kind == K_AGG else 1
        out = np.zeros((len(s), rows, DIGIT_ROW), np.int32)
        aux = np.zeros(4, np.int32)
        assert self.lib.probe_digits(kind, w, len(s), s.ctypes.data, out.ctypes.data, aux.ctypes.data) == 0
        return out, [int(v) for v in aux]


def limbs(vals, n=W):
    out = np.zeros((len(vals), n), np.uint32)
    for i, v in enumerate(vals):
        for j in range(n):
            out[i, j] = (v >> (32 * j)) & 0xffffffff
    return out


def ints(arr):
    return [sum(int(w) << (32 * j) for j, w in enumerate(row)) for row in arr]


@pytest.fixture(scope='module')
def probe_host():
    import __graft_entry__ as g
    g.build_probe(host=True)
    return Probe(g.PROBE_HOST)


@pytest.fixture(scope='module')
def probe_dev():
    import __graft_entry__ as g
    g.build_probe()
    return Probe(g.PROBE)


# ------------------------------------------------------------------------------------------------ operand catalogues
def mont_ref(a, b, p, n):
    """The exact output of a CIOS Montgomery product: (a b + m p) / R with m = -a b / p mod R, no final subtraction."""
    R = 1 << (32 * n)
    m = (-a * b * pow(p, -1, R)) % R
    return (a * b + m * p) // R


def catalogue(field, seed=0):
    """Operands over the documented domain of mul: [0, 2^13 p) for tom.p, [0, p) otherwise."""
    p, n, lazy = FIELDS[field]
    bound = (p << LAZY_BITS) if lazy else p
    rnd = random.Random(1000 + field + seed)
    v = {0, 1, 2, p - 1, p - 2, (p + 1) // 2}
    if lazy:
        v |= {p, p + 1, 2 * p - 1, 2 * p, 8 * p - 1, 8 * p, bound - 1, bound - 2}
        for k in range(LAZY_BITS + 1):
            v |= {(p << k) - 1, (p << k) + 1}
        top = (bound - 1) >> (32 * (n - 1))     # 2^15 - 1: the largest top limb below the bound
        assert top == (1 << 15) - 1
        v |= {top << (32 * (n - 1)), (top << (32 * (n - 1))) | 0xffffffff, (top << (32 * (n - 1))) - 1}
    # all-ones limb patterns below the bound
    for j in range(1, 32 * n + 1, 16):
        v.add((1 << j) - 1)
    for lo in range(n):
        for hi in range(lo, n):
            v.add(((1 << (32 * (hi - lo + 1))) - 1) << (32 * lo))
    alt = int('aa' * 4 * n, 16)
    v |= {alt, alt >> 1, int('ff00' * 2 * n, 16), int('00ff' * 2 * n, 16)}
    # low limb such that the first Montgomery quotient digit against b = 1 is 0 or 2^32 - 1
    n0 = (-pow(p, -1, 1 << 32)) % (1 << 32)
    for hi in (0, rnd.getrandbits(32 * n - 40), (bound - 1) >> 32):
        for m0 in (0, 0xffffffff):
            v.add((hi << 32) | ((m0 * pow(n0, -1, 1 << 32)) % (1 << 32)))
    for _ in range(24):
        v.add(rnd.getrandbits(rnd.randint(1, bound.bit_length())))
    return sorted(x for x in v if 0 <= x < bound)


def quotient_pairs(field, count=32, seed=0):
    """Pairs whose first quotient digit m_0 = a_0 b_0 n0' mod 2^32 is 0 or 2^32 - 1 (the all-ones carry chains)."""
    p, n, lazy = FIELDS[field]
    bound = (p << LAZY_BITS) if lazy else p
    n0 = (-pow(p, -1, 1 << 32)) % (1 << 32)
    rnd = random.Random(77 + field + seed)
    pairs = []
    while len(pairs) < count:
        a = rnd.randrange(bound) | 1
        b = rnd.randrange(bound)
        m0 = 0xffffffff if len(pairs) % 2 else 0
        b0 = (m0 * pow((a & 0xffffffff) * n0 % (1 << 32), -1, 1 << 32)) % (1 << 32) if (a & 0xffffffff) * n0 % 2 else 0
        b = (b & ~0xffffffff) | b0
        if b < bound:
            pairs.append((a, b))
    return pairs


def all_pairs(cat):
    return [x for x in cat for _ in cat], [y for _ in cat for y in cat]


# ------------------------------------------------------------------------------------------------ field checks
def check_mul(P, field, ops=(OP_MUL, OP_MUL_GENERIC)):
    p, n, lazy = FIELDS[field]
    cat = catalogue(field)
    A, B = all_pairs(cat)
    qp = quotient_pairs(field)
    A += [a for a, _ in qp]
    B += [b for _, b in qp]
    want = []
    for a, b in zip(A, B):
        t = mont_ref(a, b, p, n)
        want.append(t if lazy else (t - p if t >= p else t))
    Rinv = pow(1 << (32 * n), -1, p)
    for op in ops:
        got = P.field(field, op, A, B)
        for i, (a, b) in enumerate(zip(A, B)):
            assert got[i] == want[i], (NAMES[field], op, hex(a), hex(b), hex(got[i]), hex(want[i]))
            assert got[i] < (2 * p if lazy else p), (NAMES[field], op, hex(a), hex(b))
        assert all(g % p == a * b * Rinv % p for g, a, b in zip(got[:50], A, B))
    return len(A)


def check_linear(P, field):
    p, n, lazy = FIELDS[field]
    cat = catalogue(field)
    if lazy:
        # add: a + b exactly; sub / neg: a + 8p - b exactly for b < 8p; reduce: canonical from below 2^14 p
        A, B = all_pairs(cat)
        assert P.field(field, OP_ADD, A, B) == [a + b for a, b in zip(A, B)]
        sb = [b for b in cat if b < 8 * p]
        A2, B2 = [a for a in cat for _ in sb], [b for _ in cat for b in sb]
        assert P.field(field, OP_SUB, A2, B2) == [a + 8 * p - b for a, b in zip(A2, B2)]
        assert P.field(field, OP_NEG, sb) == [8 * p - b for b in sb]
        wide = cat + [x + (p << LAZY_BITS) for x in cat if x + (p << LAZY_BITS) < (p << (LAZY_BITS + 1))]
        assert P.field(field, OP_REDUCE, wide) == [x % p for x in wide]
        assert P.field(field, OP_IS_ZERO, wide) == [int(x % p == 0) for x in wide]
    else:
        A, B = all_pairs(cat)
        assert P.field(field, OP_ADD, A, B) == [(a + b) % p for a, b in zip(A, B)]
        assert P.field(field, OP_SUB, A, B) == [(a - b) % p for a, b in zip(A, B)]
        assert P.field(field, OP_NEG, cat) == [(-a) % p for a in cat]
        wide = cat + [x + p for x in cat if x + p < (1 << (32 * n))]
        assert P.field(field, OP_REDUCE, wide) == [x % p for x in wide]
        assert P.field(field, OP_IS_ZERO, wide) == [int(x % p == 0) for x in wide]
    eqA = cat + cat
    eqB = cat + [(x + p) if lazy and x + p < (p << LAZY_BITS) else x for x in reversed(cat)]
    assert P.field(field, OP_EQ, eqA, eqB) == [int(a % p == b % p) for a, b in zip(eqA, eqB)]


def check_mont_out(P, field):
    """from_mont and inv: canonical results from any operand of the domain; inv(0) = 0."""
    p, n, lazy = FIELDS[field]
    R = 1 << (32 * n)
    cat = catalogue(field)
    assert P.field(field, OP_FROM_MONT, cat) == [x * pow(R, -1, p) % p for x in cat]
    got = P.field(field, OP_INV, cat)
    for x, g in zip(cat, got):
        want = 0 if x % p == 0 else R * R * pow(x, -1, p) % p      # (x/R)^-1 in Montgomery form
        # strict fields: canonical; tom.p: the lazy output bound of its last product
        assert g % p == want and g < (2 * p if lazy else p), (NAMES[field], hex(x), hex(g))


@pytest.mark.parametrize('field', [0, 1, 2, 3], ids=lambda f: NAMES[f])
def test_field_edges_host(probe_host, field):
    check_mul(probe_host, field, (OP_MUL, OP_MUL_GENERIC) + ((OP_MUL_INL,) if field == 2 else ()))
    check_linear(probe_host, field)
    check_mont_out(probe_host, field)


# ------------------------------------------------------------------------------------------------ recoders
def scalar_catalogue(w):
    q, n = p256.p, p256.order
    v = {0, 1, 2, q - 1, n - 1, q - 2, n - 2, (1 << 256) - 1, 1 << 255}
    v |= {1 << b for b in range(256)}
    v |= {(1 << b) - 1 for b in range(1, 257)}
    for base in (1 << (w - 1), (1 << (w - 1)) + 1, (1 << (w - 1)) - 1, (1 << w) - 1):
        s = sum(base << (w * j) for j in range(256 // w + 1))
        v.add(s & ((1 << 256) - 1))
        v.add(s & ((1 << 255) - 1))
    for pat in ('55', 'aa', '0f', 'f0', '33', 'cc', 'ff00', '00ff'):
        v.add(int(pat * (64 // len(pat)), 16))
    rnd = random.Random(4000 + w)
    lo = 0xffffffff00000000 << 192
    v |= {rnd.randrange(lo, min(q, n)) for _ in range(12)}
    v |= {rnd.getrandbits(256) for _ in range(12)}
    return sorted(v)


def signed_digits_ref(k, w):
    """The fixed-base recoding rule: d = window + carry; d > 2^(w-1) becomes d - 2^w with a carry of 1.  The digit
    range [-2^(w-1), 2^(w-1)] admits two forms of 2^(w-1); the tables and the oracle-parity tests rely on this one."""
    half, out, carry = 1 << (w - 1), [], 0
    for j in range((256 + w) // w):
        d = ((k >> (w * j)) & ((1 << w) - 1)) + carry
        carry = int(d > half)
        out.append(d - (carry << w))
    return out


def check_signed(P, w):
    ks = scalar_catalogue(w)
    out, _ = P.digits(K_SIGNED, w, ks)
    nw = (256 + w) // w                                   # fb_windows(w)
    half = 1 << (w - 1)                                   # fb_entries(w) - 1
    for i, k in enumerate(ks):
        d = [int(x) for x in out[i, 0, :nw]]
        assert sum(dj << (w * j) for j, dj in enumerate(d)) == k, (w, hex(k))
        assert all(-half <= dj <= half for dj in d), (w, hex(k), d)
        assert out[i, 0, DIGIT_ROW - 1] == 0, (w, hex(k))  # the carry out of the last window
        assert d == signed_digits_ref(k, w), (w, hex(k))
    return out


def check_msm(P, kind):
    c, nw = (6, 43) if kind == K_MSM6 else (4, 65)
    ks = scalar_catalogue(c)
    out, _ = P.digits(kind, 0, ks)
    for i, k in enumerate(ks):
        d = [int(x) for x in out[i, 0, :nw]]
        assert sum(dj << (c * j) for j, dj in enumerate(d)) == k, (kind, hex(k))
        if kind == K_MSM6:
            assert all(-32 <= dj <= 31 for dj in d), (hex(k), d)
        else:
            assert all(-8 <= dj <= 7 for dj in d[:64]) and d[64] in (0, 1), (hex(k), d)
    return out


def check_agg(P, c):
    ks = scalar_catalogue(c)
    out, (c2, nwin, nb, ts) = P.digits(K_AGG, c, ks)
    assert (c2, nwin, nb) == (c, -(-258 // c), 1 << (c - 1))
    tb = 256 - c * (nwin - 1)
    top_max = 1 << max(tb, 0)
    assert (top_max + 1) << ts <= nb, (c, top_max, ts, nb)
    for i, k in enumerate(ks):
        d = [int(x) for x in out[i, 0, :nwin]]
        bk = [int(x) for x in out[i, 1, :nwin]]
        assert sum(dj << (c * j) for j, dj in enumerate(d)) == k, (c, hex(k))
        assert all(-(1 << (c - 1)) <= dj < (1 << (c - 1)) for dj in d[:-1]), (c, hex(k), d)
        assert 0 <= d[-1] <= top_max, (c, hex(k), d[-1])
        for j, (dj, b) in enumerate(zip(d, bk)):
            if dj == 0:
                continue
            assert 1 <= b <= nb, (c, j, dj, b)
            if j < nwin - 1:
                assert b == abs(dj)
            else:   # top window: (digit << top_shift | slot mod 2^top_shift) + 1, slot = scalar index
                assert (b - 1) >> ts == dj and (b - 1) & ((1 << ts) - 1) == i & ((1 << ts) - 1), (c, dj, b, ts)
    return out


def all_recoders(P):
    res = {}
    for w in range(2, 25):
        res[('signed', w)] = check_signed(P, w)
    res[('msm6', 6)] = check_msm(P, K_MSM6)
    res[('msm4', 4)] = check_msm(P, K_MSM4)
    for c in range(4, 17):
        res[('agg', c)] = check_agg(P, c)
    return res


def test_recoders_host(probe_host):
    all_recoders(probe_host)


# ------------------------------------------------------------------------------------------------ device
@pytest.mark.gpu
def test_field_edges_device(probe_dev, probe_host):
    """The sm_90a operations (PTX multipliers for p256.p and tom.p) on the whole catalogue: exact against Python and
    identical to the host build, op by op."""
    for field in FIELDS:
        ops = (OP_MUL, OP_MUL_GENERIC) + ((OP_MUL_INL,) if field == 2 else ())
        check_mul(probe_dev, field, ops)
        check_linear(probe_dev, field)
        check_mont_out(probe_dev, field)
        cat = catalogue(field, seed=1)
        A, B = all_pairs(cat)
        for op in range(11):
            if op == OP_MUL_INL and field != 2:
                continue
            assert probe_dev.field(field, op, A, B) == probe_host.field(field, op, A, B), (NAMES[field], op)


@pytest.mark.gpu
def test_recoders_device(probe_dev, probe_host):
    dev, host = all_recoders(probe_dev), all_recoders(probe_host)
    for key in dev:
        assert (dev[key] == host[key]).all(), key


# products compared per field by the differential check (ZKA_PROBE_DIFF_PRODUCTS overrides); on an H100 80GB HBM3,
# 2^30 took 0.08-0.13 s per field at a 700 W power limit and 0.09-0.20 s at 400 W
DIFF_PRODUCTS = int(os.environ.get('ZKA_PROBE_DIFF_PRODUCTS', str(1 << 30)))


@pytest.mark.gpu
@pytest.mark.parametrize('field', [0, 2], ids=lambda f: NAMES[f])
def test_mul_differential_device(probe_dev, field, capsys):
    """~10^9 products of hashed operands (random lengths, all-ones / zero limbs, just below the bound) for the two fields
    with a PTX multiplier (p256_mul_body, tom_mul_body): the production multiplier against the generic CIOS, plus the
    output bound.  Mismatches are re-derived in Python.  p256.n and war.p are not in it: their production mul IS
    mul_generic (war.p through a non-inlined wrapper), so only the catalogue tests against Python check them."""
    p, n, lazy = FIELDS[field]
    t0 = time.perf_counter()
    mism, bad = probe_dev.mul_diff(field, seed=0x5eed + field, count=DIFF_PRODUCTS, bound_bits=LAZY_BITS if lazy else 0)
    dt = time.perf_counter() - t0
    with capsys.disabled():
        print(f'\n[probe] {NAMES[field]}: {DIFF_PRODUCTS} products, {mism} mismatches, {dt:.2f} s')
    for a, b, r in (ints(x) for x in bad[:min(mism, 16)]):
        want = mont_ref(a, b, p, n)
        want = want if lazy else (want - p if want >= p else want)
        assert r != want or r >= (2 * p if lazy else p), 'device mismatch not confirmed in Python'
    assert mism == 0, [(hex(a), hex(b)) for a, b, _ in (ints(x) for x in bad[:min(mism, 16)])]


# ------------------------------------------------------------------------------------------------ group law
G_P256_ADD, G_P256_MADD, G_P256_DBL, G_P256_JAC_DBL, G_TOM_ADD, G_TOM_MADD, G_TOM_DBL, G_TOM_CONST = range(8)
TOM_SQRTA, TOM_D1 = 0, 2


def group_call(P, op, pairs):
    """pairs: [(P coords, Q coords)], 4 Montgomery coordinates each -> [4 coordinates] per pair."""
    import ctypes as C
    L = P.lib
    L.probe_group.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    inp = limbs([c for a, b in pairs for c in list(a) + list(b)]).reshape(len(pairs), 8, W)
    out = np.zeros((len(pairs), 4, W), np.uint32)
    assert L.probe_group(op, len(pairs), inp.ctypes.data, out.ctypes.data) == 0
    return [ints(o) for o in out]


def p256_cases():
    G = p256.generator()
    pts = [p256.identity(), G, G.neg(), G.dbl(), G.dbl().neg(), G.mul(p256.new_scalar(p256.order - 2))]
    return pts, [(a, b) for a in pts for b in pts]


def p256_affine(pt):
    """None for the identity, else canonical (x, y)"""
    q = pt.group.identity()
    q = q.add(pt)
    return None if q.to_affine() is False else (q.x, q.y)


def check_group_p256(P):
    p, R = p256.p, 1 << 256
    rnd = random.Random(5)
    mont = lambda v: v * R % p  # noqa: E731
    Rinv = pow(R, -1, p)

    def proj(pt):   # (xZ, yZ, Z) with a random Z; the identity (0 : Z : 0)
        z = rnd.randrange(1, p)
        if p256_affine(pt) is None:
            return (0, mont(z), 0, 0)
        x, y = p256_affine(pt)
        return (mont(x * z), mont(y * z), 0, mont(z))

    def got_affine(o, jac=False):
        X, Y, Z = o[0] * Rinv % p, o[1] * Rinv % p, o[3] * Rinv % p
        if Z == 0:   # the identity: (0 : Y : 0) homogeneous, (t^2 : t^3 : 0) Jacobian
            assert Y != 0 and (jac or X == 0), o
            return None
        if jac:
            return X * pow(Z * Z, -1, p) % p, Y * pow(Z * Z * Z, -1, p) % p
        return X * pow(Z, -1, p) % p, Y * pow(Z, -1, p) % p

    pts, pairs = p256_cases()
    outs = group_call(P, G_P256_ADD, [(proj(a), proj(b)) for a, b in pairs])
    for (a, b), o in zip(pairs, outs):
        assert got_affine(o) == p256_affine(a.add(b)), ('add', p256_affine(a), p256_affine(b))
    aff = [(a, b) for a, b in pairs if p256_affine(b) is not None]
    outs = group_call(P, G_P256_MADD, [(proj(a), tuple(mont(v) for v in p256_affine(b)) + (0, 0)) for a, b in aff])
    for (a, b), o in zip(aff, outs):
        assert got_affine(o) == p256_affine(a.add(b)), ('madd', p256_affine(a), p256_affine(b))
    outs = group_call(P, G_P256_DBL, [(proj(a), proj(a)) for a in pts])
    for a, o in zip(pts, outs):
        assert got_affine(o) == p256_affine(a.dbl()), ('dbl', p256_affine(a))

    def jac(pt):   # (x Z^2, y Z^3, Z); the identity (1 : 1 : 0)
        z = rnd.randrange(1, p)
        if p256_affine(pt) is None:
            return (mont(1), mont(1), 0, 0)
        x, y = p256_affine(pt)
        return (mont(x * z * z), mont(y * z * z * z), 0, mont(z))
    outs = group_call(P, G_P256_JAC_DBL, [(jac(a), jac(a)) for a in pts])
    for a, o in zip(pts, outs):
        assert got_affine(o, jac=True) == p256_affine(a.dbl()), ('jac_dbl', p256_affine(a))


def check_group_tom(P):
    """E1, the a' = 1 image of tomEdwards256 used by every variable-base addition: x' = sqrt(a) x.  Inputs carry p added
    to every coordinate (the < 2p bound of a product) and a random Z."""
    from oracle.curves import TEdwardsPoint
    p, R = tom.p, 1 << 288
    Rinv = pow(R, -1, p)
    mont = lambda v: v * R % p  # noqa: E731
    zero = [(0, 0, 0, 0)]
    s = group_call(P, G_TOM_CONST, [((TOM_SQRTA, 0, 0, 0), zero[0])])[0][0] * Rinv % p
    d1 = group_call(P, G_TOM_CONST, [((TOM_D1, 0, 0, 0), zero[0])])[0][0] * Rinv % p
    assert s * s % p == tom.a and d1 == tom.d * pow(tom.a, -1, p) % p
    G = tom.generator()
    si = pow(s, -1, p)
    T2 = TEdwardsPoint(tom, 0, p - 1)                       # order 2
    T4 = TEdwardsPoint(tom, si, 0, 0, 1)                    # order 4: image (1, 0)
    base = [tom.identity(), G, G.neg(), G.dbl(), T2, T4, T4.neg()]
    pts = base + [G.add(T2), G.add(T4), G.dbl().add(T4.neg())]
    for q in pts:
        assert tom.is_on_group(q)
    rnd = random.Random(6)

    def img(pt):   # canonical image affine (x', y)
        x, y = TEdwardsPoint(tom, pt.x, pt.y, pt.t, pt.z).to_affine()
        return s * x % p, y

    def ext(pt):
        x, y = img(pt)
        z = rnd.randrange(1, p)
        return tuple(mont(v) + p for v in (x * z, y * z, x * y * z, z))

    def got(o):
        X, Y, T, Z = (v * Rinv % p for v in o)
        assert Z != 0 and T * Z % p == X * Y % p, o
        zi = pow(Z, -1, p)
        return X * zi % p, Y * zi % p

    pairs = [(a, b) for a in pts for b in pts]
    outs = group_call(P, G_TOM_ADD, [(ext(a), ext(b)) for a, b in pairs])
    for (a, b), o in zip(pairs, outs):
        assert got(o) == img(a.add(b)), ('tom_add', img(a), img(b))

    def pre(pt):
        x, y = img(pt)
        return (mont(x), mont(y), mont(d1 * x * y % p), 0)
    outs = group_call(P, G_TOM_MADD, [(ext(a), pre(b)) for a, b in pairs])
    for (a, b), o in zip(pairs, outs):
        assert got(o) == img(a.add(b)), ('tom_madd', img(a), img(b))
    outs = group_call(P, G_TOM_DBL, [(ext(a), ext(a)) for a in pts])
    for a, o in zip(pts, outs):
        assert got(o) == img(a.dbl()), ('tom_dbl', img(a))


def test_group_law_host(probe_host):
    check_group_p256(probe_host)
    check_group_tom(probe_host)


@pytest.mark.gpu
def test_group_law_device(probe_dev):
    check_group_p256(probe_dev)
    check_group_tom(probe_dev)
