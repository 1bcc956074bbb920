"""Fixed-base tables whose windows are not all equally wide (FbShape, zk_ops.cuh): the tomEdwards256 tables g and h cover
the 257 bits of a walk in n lookups with windows of floor(257 / n) and floor(257 / n) + 1 bits, the wide ones on top.

The layout helpers and the signed-digit recoding are compared with exact Python integers; commitments, whole proofs,
verdicts and the stand-alone sub-proof entry points of a library built with a small mixed shape are compared with the
oracle, with a uniform table and with the golden fixtures; the shape a context reports is checked for ZKA_TOM_W,
ZKA_TOM_NWIN, the default, and for tables that do not fit (one lookup more)."""
import ctypes as C
import os

import numpy as np
import pytest

import common
import test_golden
import test_subproofs
from oracle.curves import tomEdwards256 as tom
from zkp_ecdsa_b200 import synth

ROW = 132
Q = tom.order


def mixed(n):
    """(w, n_lo, widths) of the shape for n lookups"""
    w = 257 // n
    n_lo = n - (257 - w * n)
    return w, n_lo, [w + (j >= n_lo) for j in range(n)]


class ShapeProbe:
    def __init__(self, path):
        self.lib = C.CDLL(path)
        self.lib.probe_shape.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        self.lib.probe_shape_digits.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def shape(self, nwin=0, uniform_w=0):
        head = np.zeros(4, np.int64)
        lay = np.zeros((ROW, 4), np.int64)
        assert self.lib.probe_shape(nwin, uniform_w, head.ctypes.data, lay.ctypes.data) == 0
        return [int(v) for v in head], lay[:int(head[1]) + 1]

    def digits(self, ks, nwin=0, uniform_w=0):
        s = np.array([[(k >> (32 * i)) & 0xffffffff for i in range(8)] for k in ks], np.uint32)
        out = np.zeros((len(ks), ROW), np.int32)
        assert self.lib.probe_shape_digits(nwin, uniform_w, len(ks), s.ctypes.data, out.ctypes.data) == 0
        return out


def scalars(widths, seed):
    """0, 1, the largest values, patterns that carry through every window, a value whose top window receives only the
    carry, and random ones"""
    pos = [sum(widths[:j]) for j in range(len(widths) + 1)]
    half_all = sum(1 << (p + w - 1) for p, w in zip(pos[:-1], widths) if p + w - 1 < 256)   # every window at its half
    top = pos[-2]
    d = synth.Drbg(seed, 'shape')
    ks = [0, 1, (1 << 256) - 1, Q - 1, Q, int('55' * 32, 16), int('aa' * 32, 16), half_all, (half_all + 1) & ((1 << 256) - 1),
          (1 << top) - 1,                      # all ones below the top window: it gets the carry and nothing else
          (1 << top) - (1 << (top - 1)) + 1,   # the window below the top one just above its half
          1 << top, (1 << 255) + 1]
    return [k & ((1 << 256) - 1) for k in ks] + [int.from_bytes(d.bytes(32), 'big') for _ in range(40)]


def check_layout(pr):
    assert pr.shape(11)[0] == [23, 11, 7, 257] and pr.shape(12)[0] == [21, 12, 7, 257]
    assert int(pr.shape(11)[1][11, 3]) == 7 * ((1 << 22) + 1) + 4 * ((1 << 23) + 1)
    for n in (11, 12, 13, 27, 37, 64, 128):
        w, n_lo, widths = mixed(n)
        head, lay = pr.shape(n)
        assert head == [w, n, n_lo, 257] and sum(widths) == 257 and max(widths) <= 24
        ent = [(1 << (x - 1)) + 1 for x in widths]
        assert [int(v) for v in lay[:n, 0]] == widths and [int(v) for v in lay[:n, 2]] == ent
        assert [int(v) for v in lay[:, 1]] == [sum(widths[:j]) for j in range(n + 1)]
        assert [int(v) for v in lay[:, 3]] == [sum(ent[:j]) for j in range(n + 1)]
    for w in (2, 8, 13, 22, 24):   # a uniform table: (256 + w) // w windows of w bits at j w, as before
        n = (256 + w) // w
        head, lay = pr.shape(uniform_w=w)
        assert head == [w, n, n, n * w]
        assert [int(v) for v in lay[:, 1]] == [j * w for j in range(n + 1)]
        assert [int(v) for v in lay[:, 3]] == [j * ((1 << (w - 1)) + 1) for j in range(n + 1)]
    assert pr.lib.probe_shape(10, 0, None, None) == -1 and pr.lib.probe_shape(129, 0, None, None) == -1


def check_recoding(pr, seed):
    for n, uw in ((11, 0), (12, 0), (27, 0), (37, 0), (128, 0), (0, 13), (0, 16)):
        widths = [uw] * ((256 + uw) // uw) if uw else mixed(n)[2]
        pos = [sum(widths[:j]) for j in range(len(widths))]
        ks = scalars(widths, seed + n + uw)
        out = pr.digits(ks, n, uw)
        for k, row in zip(ks, out):
            ds = [int(v) for v in row[:len(widths)]]
            assert sum(d << p for d, p in zip(ds, pos)) == k, (n, uw, hex(k))
            assert all(abs(d) <= 1 << (w - 1) for d, w in zip(ds, widths)), (n, uw, hex(k))
            assert row[ROW - 1] == 0 and not row[len(widths):ROW - 1].any()
        assert [int(v) for v in out[9][:len(widths)]] == [-1] + [0] * (len(widths) - 2) + [1]   # all ones below the top window


def load(path_or_none, **env):
    """a library (hostsim by path, the product on cuda:0 otherwise) created under the given ZKA_* settings only"""
    keys = ('ZKA_TOM_W', 'ZKA_TOM_NWIN', 'ZKA_TOM_TABLE_MAX', 'ZKA_P256_HW')
    old = {k: os.environ.pop(k, None) for k in keys}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        from zkp_ecdsa_b200.capi import ZkaLib
        return ZkaLib(path_or_none) if path_or_none else ZkaLib(device=0)
    finally:
        for k in keys:
            os.environ.pop(k, None)
            if old[k] is not None:
                os.environ[k] = old[k]


def table_bytes(n):
    return 128 * sum((1 << (w - 1)) + 1 for w in mixed(n)[2])


@pytest.fixture(scope='module')
def host_path():
    import __graft_entry__ as g
    g.build_hostsim()
    return g.HOSTSIM


@pytest.fixture(scope='module')
def mixed27(host_path):
    """hostsim with 27 lookups: 13 windows of 9 bits below 14 of 10"""
    L = load(host_path, ZKA_TOM_NWIN=27, ZKA_P256_HW=8)
    cfg = L.config()
    assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo'], cfg['tom_fallback']) == (9, 27, 13, False)
    return L


def walk_scalars(widths, seed):
    """values and blinders at the ends of a walk and at the step from the narrow to the wide windows"""
    pos = [sum(widths[:j]) for j in range(len(widths) + 1)]
    d = synth.Drbg(seed, 'shape-walk')
    n_lo = widths.index(max(widths)) if max(widths) != min(widths) else len(widths)
    vs = [0, 1, Q - 1, 1 << (widths[0] - 1), (1 << widths[0]) - 1, d.below(1 << (pos[-2] - 1)), (1 << pos[-2]) - 1]
    if n_lo < len(widths):
        b = pos[n_lo]   # first wide window: its half-range digit, a carry into it, all ones across the step
        vs += [1 << (b + widths[n_lo] - 1), (1 << b) - 1, ((1 << (b + widths[n_lo])) - 1) ^ ((1 << pos[n_lo - 1]) - 1)]
    vs = [v % Q for v in vs] + [d.below(Q) for _ in range(3)]
    return [v for v in vs for _ in vs], [r for _ in vs for r in vs]


def check_commits(L, seed, uniform=None):
    """v g + r h from the library's tables against the oracle (and a library with uniform tables)"""
    cfg = L.config()
    widths = [cfg['tom_w'] + (j >= cfg['tom_n_lo']) for j in range(cfg['tom_nwin'])]
    P, po = common.make_params(L, seed, 16)
    vs, rs = walk_scalars(widths, seed)
    out = L.tom_commit_batch(P, common.be(vs, 32), common.be(rs, 32))
    g = common.pg(L)
    for i in range(0, len(vs), 5):
        e = po.ProofGroup.h.dblmul(g.new_scalar(rs[i]), po.ProofGroup.g, g.new_scalar(vs[i])).to_bytes()
        assert out[i].tobytes() == e, (i, hex(vs[i]), hex(rs[i]))
    if uniform is not None:
        Pu, _ = common.make_params(uniform, seed, 16)
        assert (uniform.tom_commit_batch(Pu, common.be(vs, 32), common.be(rs, 32)) == out).all()
        uniform.params_destroy(Pu)
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------------- host build
def test_shape_layout_and_recoding_host():
    import __graft_entry__ as g
    g.build_probe_shape(host=True)
    pr = ShapeProbe(g.PROBE_SHAPE_HOST)
    check_layout(pr)
    check_recoding(pr, seed=1)


def test_mixed_shape_commitments_host(mixed27, hostsim):
    check_commits(mixed27, seed=11, uniform=hostsim)


@pytest.mark.parametrize('tag', ['a', 'b', 'c', 'd'])
def test_mixed_shape_matches_golden_host(mixed27, tag):
    test_golden._check_lib(mixed27, tag)


def test_mixed_shape_proofs_and_verdicts_host(mixed27):
    common.check_prove_parity(mixed27, B=2, N=5, sec_level=16, seed=12, make_tape=synth.edge_tape)
    common.check_verify_parity(mixed27, N=5, sec_level=20, seed=13, tampers=8)


def test_mixed_shape_subproofs_host(mixed27):
    for kind in ('equality', 'mult', 'pointadd'):
        test_subproofs.check_prove_small(mixed27, kind, seed=14, B=2)
        test_subproofs.check_verify_small(mixed27, kind, seed=15, tampers=2)
    test_subproofs.check_prove_exp(mixed27, sec=8, with_q=True, seed=16, B=1)
    test_subproofs.check_verify_exp(mixed27, sec=8, K=8, with_q=False, seed=17, tampers=2)
    test_subproofs.check_prove_membership(mixed27, [3, 5, 7, 11, 13], [3, 0], seed=18)
    test_subproofs.check_verify_membership(mixed27, [3, 5, 7, 11, 13], 3, seed=19, tampers=2)


def test_mixed_shape_37_lookups_host(host_path):
    """2 windows of 6 bits below 35 of 7: only two narrow windows"""
    L = load(host_path, ZKA_TOM_NWIN=37, ZKA_P256_HW=8)
    cfg = L.config()
    assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo']) == (6, 37, 2)
    check_commits(L, seed=21)
    common.check_prove_parity(L, B=1, N=4, sec_level=16, seed=22)


def test_reported_shape_host(host_path):
    L = load(host_path, ZKA_TOM_W=11, ZKA_TOM_NWIN=27, ZKA_P256_HW=8)   # a pinned width wins: the uniform table
    cfg = L.config()
    assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo'], cfg['tom_fallback']) == (11, 24, 24, False)
    L = load(host_path, ZKA_TOM_NWIN=200, ZKA_TOM_W=10, ZKA_P256_HW=8)
    assert (L.config()['tom_w'], L.config()['tom_nwin']) == (10, 26)


def test_tables_that_do_not_fit_host(host_path):
    """a table above ZKA_TOM_TABLE_MAX is an allocation that failed: one lookup more, reported; a pinned width and a
    limit below the smaller table fail instead"""
    from zkp_ecdsa_b200.capi import ZkaError
    assert table_bytes(28) < table_bytes(27)
    L = load(host_path, ZKA_TOM_NWIN=27, ZKA_TOM_TABLE_MAX=table_bytes(27) - 1, ZKA_P256_HW=8)
    cfg = L.config()
    assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo'], cfg['tom_fallback']) == (9, 28, 23, True)
    check_commits(L, seed=31)
    L = load(host_path, ZKA_TOM_NWIN=27, ZKA_TOM_TABLE_MAX=table_bytes(27), ZKA_P256_HW=8)
    assert L.config()['tom_nwin'] == 27 and not L.config()['tom_fallback']
    with pytest.raises(ZkaError):
        load(host_path, ZKA_TOM_NWIN=27, ZKA_TOM_TABLE_MAX=table_bytes(28) - 1, ZKA_P256_HW=8)
    with pytest.raises(ZkaError):
        load(host_path, ZKA_TOM_W=9, ZKA_TOM_TABLE_MAX=1000, ZKA_P256_HW=8)


# ------------------------------------------------------------------------------------------------- device
@pytest.mark.gpu
def test_shape_layout_and_recoding_device():
    import __graft_entry__ as g
    g.build_probe_shape()
    pr = ShapeProbe(g.PROBE_SHAPE)
    check_layout(pr)
    check_recoding(pr, seed=2)


@pytest.mark.gpu
def test_default_shape_device(gpu_engine):
    """the default: 11 lookups, 7 windows of 23 bits below 4 of 24; its commitments at the walk ends and the width step"""
    cfg = gpu_engine.lib.config()
    if cfg['tom_fallback']:
        assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo']) == (21, 12, 7)
        pytest.skip('the card had no room for the 11-lookup tables')
    assert (cfg['tom_w'], cfg['tom_nwin'], cfg['tom_n_lo']) == (23, 11, 7)
    check_commits(gpu_engine.lib, seed=41)


@pytest.mark.gpu
def test_mixed_shape_device():
    """a small mixed shape on the device against the oracle, a uniform table, a golden case and whole proofs"""
    L = load(None, ZKA_TOM_NWIN=27, ZKA_P256_HW=11)
    U = load(None, ZKA_TOM_W=14, ZKA_P256_HW=11)
    try:
        assert (L.config()['tom_w'], L.config()['tom_nwin'], L.config()['tom_n_lo']) == (9, 27, 13)
        check_commits(L, seed=42, uniform=U)
        test_golden._check_lib(L, 'a')
        common.check_prove_parity(L, B=3, N=9, sec_level=16, seed=43, make_tape=synth.edge_tape)
        common.check_verify_parity(L, N=6, sec_level=20, seed=44, tampers=8)
        test_subproofs.check_prove_small(L, 'pointadd', seed=45, B=2)
        test_subproofs.check_verify_small(L, 'mult', seed=46, tampers=2)
    finally:
        L.close()
        U.close()
