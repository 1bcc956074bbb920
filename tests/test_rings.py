"""Ring sets: one prove / verify call over rows that each name their own ring (include/zkattest.h, "ring sets").

Every row's proof bytes, verdict and status must be those of the one-ring call with that row's ring, so the oracle
(oracle/zkattest.py, oracle/cpu) applies row by row: on the host simulator (both proof groups) and on the GPU.
"""
import ctypes as C

import numpy as np
import pytest

import common
from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from zkp_ecdsa_b200 import api, synth
from zkp_ecdsa_b200 import verify_tape as VT

SIZES = [2, 5, 6, 8, 17]                  # depths 1, 3, 3, 3, 5
RING_OF = [3, 0, 1, 2, 2, 4, 1, 0]        # runs of depth 3 | 1 | 3 3 3 | 5 | 3 | 1


def _seeds(rows, tag):
    return np.frombuffer(synth.Drbg(rows, f'rings-seeds-{tag}').bytes(32 * rows), np.uint8).reshape(rows, 32).copy()


def _n(N):
    return VT.ceil_log2(N)


class Set:
    """A zka_rings handle of a library object, destroyed by close()."""

    def __init__(self, L, wl):
        self.L, self.sizes = L, wl.sizes
        self.h = L.rings_create(np.array(wl.sizes, np.uint32), wl.keys)

    def close(self):
        self.L.rings_destroy(self.h)


def prove_rings(L, P, rs, wl, tape, S, ring_of=None, which=None):
    ring_of = wl.ring_of if ring_of is None else ring_of
    which = wl.which if which is None else which
    B = wl.B
    ps = L.proof_max_len(max(wl.sizes[r] for r in ring_of), S)
    proofs, plen, st = np.zeros((B, ps), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)
    L.prove_batch_rings(P, rs.h, np.ascontiguousarray(ring_of, np.uint32), B, wl.msg_hash, wl.sig, wl.pk,
                        np.ascontiguousarray(which, np.uint32), tape, tape.shape[1], proofs, ps, plen, st)
    return proofs, plen, st


def prove_rings_seeded(L, P, rs, wl, seeds, S):
    B = wl.B
    ps = L.proof_max_len(max(wl.sizes), S)
    proofs, plen, st = np.zeros((B, ps), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)
    L.prove_batch_rings_seeded(P, rs.h, wl.ring_of, B, wl.msg_hash, wl.sig, wl.pk, wl.which, seeds, proofs, ps, plen, st)
    return proofs, plen, st


def verify_rings(L, P, rs, ring_of, msg, proofs, plen, vt, K):
    B = msg.shape[0]
    ok, st = np.zeros(B, np.uint8), np.zeros(B, np.int32)
    L.verify_batch_rings(P, rs.h, np.ascontiguousarray(ring_of, np.uint32), B, msg, proofs, proofs.shape[1], plen, vt, vt.shape[1],
                         K, ok, st)
    return ok, st


def row_verify_tape(sizes, ring_of, S, K, seed):
    """Each row's verify tape laid out for its own ring size, all at the stride of the largest ring used."""
    stride = VT.verify_tape_len(max(sizes[r] for r in ring_of), K)
    return np.concatenate([VT.random_verify_tape(1, stride, sizes[r], S, seed=seed + b) for b, r in enumerate(ring_of)])


def row_seed_tape(L, kind, seeds, sizes, ring_of, S, K=0):
    """zka_seed_tape of each row with its own ring size, at the stride of the largest ring used."""
    Nmax = max(sizes[r] for r in ring_of)
    stride = L.prove_tape_len(Nmax, S) if kind == 0 else L.verify_tape_len_ex(Nmax, S, K)
    out = np.zeros((len(ring_of), stride), np.uint8)
    for b, r in enumerate(ring_of):
        t = L.seed_tape(kind, seeds[b:b + 1].copy(), sizes[r], S, K)
        out[b, :t.shape[1]] = t[0]
    return out


def oracle_row(po, wl, b, tape_row, r=None):
    r = int(wl.ring_of[b]) if r is None else r
    tp = Tape(tape_row)
    pr = OZ.prove_signature_list(po, wl.msg_hash[b].tobytes(), wl.sig[b].tobytes(), wl.pk[b].tobytes(), int(wl.which[b]),
                                 wl.ring_ints(r), tp)
    return pr, tp


# ------------------------------------------------------------------------------------------------ prove vs the oracle
def check_prove_parity(L, sizes=SIZES, ring_of=RING_OF, S=16, seed=91):
    P, po = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(ring_of), sizes, ring_of, seed=seed)
    rs = Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(sizes), S), seed=seed + 100)
    proofs, plen, st = prove_rings(L, P, rs, wl, tape, S)
    assert (st == 0).all(), st
    for b in range(wl.B):
        pr, tp = oracle_row(po, wl, b, tape[b].tobytes())
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), f'row {b} (ring {wl.ring_of[b]}) differs from the oracle'
        z = sum(1 for e in pr.expProof if e.alpha is None)
        n = _n(sizes[wl.ring_of[b]])
        assert tp.calls == 3 + 4 * S + 40 * z + 5 * n
        assert plen[b] == flat.proof_len(z, n, S)
    # the same rows in another order give the same bytes
    perm = np.random.default_rng(seed).permutation(wl.B)
    sub = _rows(wl, perm)
    p2, l2, s2 = prove_rings(L, P, rs, sub, tape[perm].copy(), S)
    assert (s2 == 0).all()
    for i, b in enumerate(perm):
        assert p2[i, :l2[i]].tobytes() == proofs[b, :plen[b]].tobytes(), (i, b)
    rs.close()
    L.params_destroy(P)
    return wl, proofs, plen


def _rows(wl, idx):
    """The rows `idx` of a RingsWorkload, as a workload of their own over the same rings."""
    sub = synth.RingsWorkload.__new__(synth.RingsWorkload)
    sub.__dict__.update(wl.__dict__)
    sub.B = len(idx)
    for k in ('msg_hash', 'sig', 'pk', 'which', 'ring_of'):
        setattr(sub, k, getattr(wl, k)[np.asarray(idx)].copy())
    return sub


def test_rings_prove_matches_oracle_hostsim(hostsim):
    check_prove_parity(hostsim)


def test_rings_prove_matches_oracle_hostsim_s80(hostsim):
    check_prove_parity(hostsim, sizes=[5, 17], ring_of=[1], S=80, seed=92)


def test_rings_prove_matches_oracle_hostsim_war(hostsim_war):
    check_prove_parity(hostsim_war, sizes=[2, 5, 17], ring_of=[2, 1, 1, 0], S=16, seed=93)


def test_rings_pad_with_their_own_first_entry(hostsim):
    """Rings of 5 and 17 entries are padded with their own first entry: every row equals a one-ring zka_prove_batch of
    its ring, whose padding is that ring's first entry, and the set's first ring has another first entry."""
    L, S, seed = hostsim, 16, 94
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(4, [6, 5, 17], [1, 2, 1, 2], seed=seed)
    assert wl.rings[0][0].tobytes() not in (wl.rings[1][0].tobytes(), wl.rings[2][0].tobytes())
    rs = Set(L, wl)
    tape = synth.random_tape(4, L.prove_tape_len(17, S), seed=seed)
    proofs, plen, st = prove_rings(L, P, rs, wl, tape, S)
    assert (st == 0).all()
    for r in (1, 2):
        rows = np.flatnonzero(wl.ring_of == r)
        one = synth.Workload.__new__(synth.Workload)
        one.B, one.N, one.ring = len(rows), wl.sizes[r], wl.rings[r]
        one.msg_hash, one.sig, one.pk, one.which = (getattr(wl, k)[rows].copy() for k in ('msg_hash', 'sig', 'pk', 'which'))
        rp, rl, rst = common.run_prove(L, P, one, tape[rows].copy(), S)
        assert (rst == 0).all()
        for i, b in enumerate(rows):
            assert proofs[b, :plen[b]].tobytes() == rp[i, :rl[i]].tobytes(), (r, b)
    rs.close()
    L.params_destroy(P)


def test_rings_seeded_prove_equals_tape_prove_hostsim(hostsim):
    L, S, seed = hostsim, 16, 95
    P, po = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(RING_OF), SIZES, RING_OF, seed=seed)
    rs = Set(L, wl)
    seeds = _seeds(wl.B, f'p{seed}')
    proofs, plen, st = prove_rings_seeded(L, P, rs, wl, seeds, S)
    assert (st == 0).all(), st
    tape = row_seed_tape(L, 0, seeds, SIZES, wl.ring_of, S)
    tp, tl, ts = prove_rings(L, P, rs, wl, tape, S)
    assert (ts == 0).all() and np.array_equal(tl, plen)
    for b in range(wl.B):
        assert proofs[b, :plen[b]].tobytes() == tp[b, :tl[b]].tobytes(), b
    pr, _ = oracle_row(po, wl, 5, tape[5].tobytes())
    assert proofs[5, :plen[5]].tobytes() == flat.ser_proof(pr)
    rs.close()
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------------------ R = 1
def test_rings_one_ring_equals_the_one_ring_calls_hostsim(hostsim):
    L, S, K, N, seed = hostsim, 16, 5, 6, 96
    P, _ = common.make_params(L, seed, S)
    wl = synth.Workload(B=4, N=N, seed=seed)
    rw = synth.RingsWorkload.__new__(synth.RingsWorkload)
    rw.B, rw.sizes, rw.keys, rw.ring_of = 4, [N], wl.ring, np.zeros(4, np.uint32)
    rw.msg_hash, rw.sig, rw.pk = wl.msg_hash, wl.sig, wl.pk
    rs = Set(L, rw)
    which = wl.which.copy()
    which[2] = N                        # outside the ring: a row status
    tape = synth.random_tape(4, L.prove_tape_len(N, S), seed=seed)
    proofs, plen, st = prove_rings(L, P, rs, rw, tape, S, which=which)
    one = synth.Workload.__new__(synth.Workload)
    one.__dict__.update(wl.__dict__)
    one.which = which
    rp, rl, rst = common.run_prove(L, P, one, tape, S)
    assert np.array_equal(st, rst) and st[2] == 6 and np.array_equal(plen, rl) and np.array_equal(proofs, rp)
    vt = VT.random_verify_tape(4, L.verify_tape_len_ex(N, S, K), N, S, seed=seed)
    bad = proofs.copy()
    bad[1, 400] ^= 1
    msg = wl.msg_hash.copy()
    msg[3, 0] ^= 1
    for pr in (proofs, bad):
        ok, vst = verify_rings(L, P, rs, rw.ring_of, msg, pr, plen, vt, K)
        ok2, vst2 = np.zeros(4, np.uint8), np.zeros(4, np.int32)
        L.verify_batch_ex(P, 4, msg, wl.ring, N, pr, pr.shape[1], plen, vt, vt.shape[1], ok2, vst2, K)
        assert np.array_equal(ok, ok2) and np.array_equal(vst, vst2), (ok, ok2, vst, vst2)
    assert list(ok) == [1, 0, 0, 0]
    rs.close()
    L.params_destroy(P)


# -------------------------------------------------------------------------------------------------- verify
def check_verify_parity(L, S=16, K=5, seed=97, tampers=8):
    P, po = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(RING_OF), SIZES, RING_OF, seed=seed)
    rs = Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(SIZES), S), seed=seed)
    proofs, plen, st = prove_rings(L, P, rs, wl, tape, S)
    assert (st == 0).all()
    vt = row_verify_tape(SIZES, wl.ring_of, S, K, seed)
    passed = L.stat('agg_pass')
    ok, vst = verify_rings(L, P, rs, wl.ring_of, wl.msg_hash, proofs, plen, vt, K)
    assert ok.all() and not vst.any(), (ok, vst)
    assert L.stat('agg_pass') > passed
    # tampered rows, and rows verified against another ring of the same depth (6 -> 8) or of another depth (6 -> 2, 17)
    rng = np.random.default_rng(seed)
    cases = []                                            # (row, proof bytes, msg, ring)
    for k in range(tampers):
        b = int(rng.integers(0, wl.B))
        p, msg = proofs[b, :plen[b]].copy(), wl.msg_hash[b].copy()
        kind = k % 4
        if kind == 0:
            p[int(rng.integers(0, len(p)))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:
            p = p[:len(p) - 1 - int(rng.integers(0, 40))]
        elif kind == 2:
            p[len(p) - 1 - getattr(L, 'ws', 33) * int(rng.integers(0, 5))] ^= 1
        else:
            msg[int(rng.integers(0, 32))] ^= 1
        cases.append((b, p, msg, int(wl.ring_of[b])))
    b6 = int(np.flatnonzero(wl.ring_of == 2)[0])
    for other in (3, 0, 4):
        cases.append((b6, proofs[b6, :plen[b6]].copy(), wl.msg_hash[b6].copy(), other))
    T = len(cases)
    ring_of = np.array([c[3] for c in cases], np.uint32)
    vt2 = row_verify_tape(SIZES, ring_of, S, K, seed + 50)
    arr = np.zeros((T, proofs.shape[1]), np.uint8)
    lens = np.zeros(T, np.uint32)
    msgs = np.zeros((T, 32), np.uint8)
    for i, (_, p, m, _) in enumerate(cases):
        arr[i, :len(p)] = p
        lens[i] = len(p)
        msgs[i] = m
    ok, vst = verify_rings(L, P, rs, ring_of, msgs, arr, lens, vt2, K)
    verdicts = []
    for i, (_, p, m, r) in enumerate(cases):
        try:
            prf = flat.de_proof(p.tobytes(), S)
            exp = OZ.verify_signature_list(po, m.tobytes(), wl.ring_ints(r), prf,
                                           Tape(VT.oracle_stream(vt2[i].tobytes(), SIZES[r], S)), K)
        except ValueError:
            exp = 'err'
        got = 'err' if vst[i] else bool(ok[i])
        assert got == exp, (i, got, int(vst[i]), exp)
        verdicts.append(got)
    assert verdicts[-3:] == [False, False, False]
    # seeded verification equals the tape call on each row's own expansion
    seeds = _seeds(T, f'v{seed}')
    oks, sts = np.zeros(T, np.uint8), np.zeros(T, np.int32)
    L.verify_batch_rings_seeded(P, rs.h, ring_of, T, msgs, arr, arr.shape[1], lens, seeds, K, oks, sts)
    vt3 = row_seed_tape(L, 1, seeds, SIZES, ring_of, S, K)
    ok3, st3 = verify_rings(L, P, rs, ring_of, msgs, arr, lens, vt3, K)
    assert np.array_equal(oks, ok3) and np.array_equal(sts, st3)
    rs.close()
    L.params_destroy(P)


def test_rings_verify_matches_oracle_hostsim(hostsim):
    check_verify_parity(hostsim)


def test_rings_verify_matches_oracle_hostsim_war(hostsim_war):
    check_verify_parity(hostsim_war, seed=98, tampers=4)


# ----------------------------------------------------------------------------------------------- argument checks
def test_rings_argument_checks(hostsim):
    L, S, seed = hostsim, 16, 99
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(3, [5, 17], [0, 1, 0], seed=seed)
    lib, ctx = L.lib, L.ctx
    p = C.c_void_p
    ptr = lambda a: p(a.ctypes.data)   # noqa: E731
    h = p()
    keys = np.zeros(((1 << 20) + 1, 32), np.uint8)
    for sizes in ([1], [5, 1], [(1 << 20) + 1], [8, (1 << 20) + 1]):
        s = np.array(sizes, np.uint32)
        assert lib.zka_rings_create(ctx, s.size, ptr(s), ptr(keys), C.byref(h)) == -1, sizes
    s = np.array([5], np.uint32)
    assert lib.zka_rings_create(ctx, 0, ptr(s), ptr(keys), C.byref(h)) == -1
    assert lib.zka_rings_create(ctx, 1, ptr(s), p(0), C.byref(h)) == -1
    s = np.array([1 << 20] * 17, np.uint32)                 # 17 * 2^20 padded entries > 2^24
    assert lib.zka_rings_create(ctx, s.size, ptr(s), ptr(keys), C.byref(h)) == -1
    assert lib.zka_rings_create(ctx, 0xffffffff, ptr(s), ptr(keys), C.byref(h)) == -1   # refused before sizes is read
    rs = Set(L, wl)
    tape = synth.random_tape(3, L.prove_tape_len(17, S), seed=seed)
    ps = L.proof_max_len(17, S)
    proofs, plen, st = np.zeros((3, ps), np.uint8), np.zeros(3, np.uint32), np.zeros(3, np.int32)
    ok = np.zeros(3, np.uint8)
    vt = row_verify_tape(wl.sizes, wl.ring_of, S, 5, seed)

    def prove(handle, ring_of, B=3, which=wl.which, stride=ps, tstride=tape.shape[1]):
        return lib.zka_prove_batch_rings(ctx, P, handle, ptr(ring_of), B, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(which),
                                         ptr(tape), tstride, ptr(proofs), stride, ptr(plen), ptr(st))

    def verify(handle, ring_of, B=3):
        return lib.zka_verify_batch_rings(ctx, P, handle, ptr(ring_of), B, ptr(wl.msg_hash), ptr(proofs), ps, ptr(plen), ptr(vt),
                                          vt.shape[1], 5, ptr(ok), ptr(st))
    bad = np.array([0, 2, 1], np.uint32)
    st[:] = 77
    assert prove(rs.h, bad) == -1 and verify(rs.h, bad) == -1
    assert (st == 77).all()                                 # nothing ran
    assert prove(p(0), wl.ring_of) == -1 and verify(p(0), wl.ring_of) == -1
    assert prove(rs.h, wl.ring_of, B=0) == 0 and verify(rs.h, wl.ring_of, B=0) == 0
    assert prove(rs.h, wl.ring_of, stride=L.proof_max_len(5, S)) == -1      # strides cover the largest ring used
    assert prove(rs.h, wl.ring_of, tstride=32 * (3 + 4 * S + 5 * 5) - 32) == -1   # the draws before any item, n = 5
    # which = 5 in a ring of 5 and which = 6 (inside its padding to 8) are row statuses; the ring of 17 takes 5
    which = np.array([5, 5, 6], np.uint32)
    assert prove(rs.h, wl.ring_of, which=which) == 0
    assert list(st) == [6, 0, 6], st
    rs.close()
    L.params_destroy(P)


def test_engine_ring_set_api(hostsim, monkeypatch):
    """api.Engine.load_rings / prove_batch_rings[_seeded] / verify_batch_rings[_seeded] against the oracle."""
    eng = api.Engine.__new__(api.Engine)
    eng.lib, eng.proof_group = hostsim, hostsim.group
    P, po = common.make_params(hostsim, 100, 20)

    class Params:
        handle, sec_level = P, 20
    wl = synth.RingsWorkload(3, [5, 6, 17], [2, 0, 2], seed=100)
    rings = eng.load_rings([wl.ring_ints(0), wl.rings[1], wl.ring_ints(2)])
    assert rings.sizes == [5, 6, 17] and rings.depths == [3, 3, 5]
    tape = synth.random_tape(3, hostsim.prove_tape_len(17, 20), seed=100)
    res = eng.prove_batch_rings(Params, rings, wl.ring_of, wl.msg_hash, wl.sig, wl.pk, wl.which, tape)
    assert (res.status == 0).all() and res.proofs.shape[1] == hostsim.proof_max_len(17, 20)
    pr, _ = oracle_row(po, wl, 1, tape[1].tobytes())
    assert res.proof_bytes(1) == flat.ser_proof(pr)
    vt = row_verify_tape(wl.sizes, wl.ring_of, 20, 20, 100)
    ok, st = eng.verify_batch_rings(Params, rings, wl.ring_of, wl.msg_hash, res.proofs, res.proof_len, vt)
    assert ok.all() and not st.any()
    drawn = []
    real = api.os.urandom
    monkeypatch.setattr(api.os, 'urandom', lambda n: drawn.append(real(n)) or drawn[-1])
    rs = eng.prove_batch_rings_seeded(Params, rings, wl.ring_of, wl.msg_hash, wl.sig, wl.pk, wl.which)
    ok, st = eng.verify_batch_rings_seeded(Params, rings, wl.ring_of, wl.msg_hash, rs.proofs, rs.proof_len, samples=5)
    monkeypatch.undo()
    assert [len(d) for d in drawn] == [96, 96]
    assert (rs.status == 0).all() and ok.all() and not st.any()
    with pytest.raises(ValueError):
        rings.largest([3])
    rings.close()
    rings.close()
    hostsim.params_destroy(P)


# ------------------------------------------------------------------------------------------------------------- GPU
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_ring_of(n8, big, seed):
    """n8 rings of 8 with one row each (in a shuffled order), then the rows of the `big` rings in runs of 100."""
    ro = list(np.random.default_rng(seed).permutation(n8))
    left = dict(big)
    while any(left.values()):
        for r in left:
            t = min(100, left[r])
            ro += [r] * t
            left[r] -= t
    return np.array(ro, np.uint32)


def _one_ring(wl, rows, r):
    one = synth.Workload.__new__(synth.Workload)
    one.B, one.N, one.ring = len(rows), wl.sizes[r], wl.rings[r]
    one.msg_hash, one.sig, one.pk, one.which = (getattr(wl, k)[rows].copy() for k in ('msg_hash', 'sig', 'pk', 'which'))
    return one


def check_gpu_rings(L, n8, big_sizes, rows_big, S, seed, K=20):
    import torch
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    sizes = [8] * n8 + list(big_sizes)
    ring_of = gpu_ring_of(n8, [(n8 + i, rows_big) for i in range(len(big_sizes))], seed)
    B = len(ring_of)
    P, po = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(B, sizes, ring_of, seed=seed)
    rs = Set(L, wl)
    Nmax = max(sizes)
    tape = synth.random_tape(B, L.prove_tape_len(Nmax, S), seed=seed + 1)
    ps = L.proof_max_len(Nmax, S)
    # the only route without ring sets: one zka_prove_batch / zka_verify_batch_ex per ring
    ref = np.zeros((B, ps), np.uint8)
    rlen, rst = np.zeros(B, np.uint32), np.zeros(B, np.int32)
    by_ring = [np.flatnonzero(ring_of == r) for r in range(len(sizes))]
    for r, rows in enumerate(by_ring):
        one = _one_ring(wl, rows, r)
        t = tape[rows][:, :L.prove_tape_len(sizes[r], S)].copy()
        p, ln, s = common.run_prove(L, P, one, t, S)
        ref[rows, :p.shape[1]], rlen[rows], rst[rows] = p, ln, s
    assert (rst == 0).all()
    cfg = L.config()
    try:
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            for chunk in (None, 128):
                if chunk:
                    L.set_option('chunk', chunk)
                    L.set_option('host_chunk', chunk)
                proofs, plen, st = prove_rings(L, P, rs, wl, tape, S)
                assert (st == 0).all() and np.array_equal(plen, rlen), ('host', lanes, chunk)
                assert all(proofs[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes() for b in range(B)), ('host', lanes, chunk)
                dp = torch.zeros(B * ps, dtype=torch.uint8, device='cuda')
                dl = torch.zeros(B, dtype=torch.int32, device='cuda')
                ds = torch.zeros(B, dtype=torch.int32, device='cuda')
                dro, dm, dsig, dpk, dw, dt = (_dev(x) for x in (ring_of.view(np.int32), wl.msg_hash, wl.sig, wl.pk,
                                                                 wl.which.view(np.int32), tape))
                L.prove_batch_rings(P, rs.h, dro.data_ptr(), B, dm.data_ptr(), dsig.data_ptr(), dpk.data_ptr(), dw.data_ptr(),
                                    dt.data_ptr(), tape.shape[1], dp.data_ptr(), ps, dl.data_ptr(), ds.data_ptr())
                torch.cuda.synchronize()
                assert not ds.cpu().numpy().any()
                assert np.array_equal(dl.cpu().numpy().view(np.uint32), rlen), ('device', lanes, chunk)
                got = dp.cpu().numpy().reshape(B, ps)
                assert all(got[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes() for b in range(B)), ('device', lanes, chunk)
                L.set_option('chunk', cfg['chunk'])
                L.set_option('host_chunk', 2048)
        # verification: verdicts and statuses of the per-ring calls; an all-valid mixed-ring chunk passes the aggregate
        vt = row_verify_tape(sizes, ring_of, S, K, seed)
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            passed = L.stat('agg_pass')
            ok, vst = verify_rings(L, P, rs, ring_of, wl.msg_hash, ref, rlen, vt, K)
            assert ok.all() and not vst.any()
            assert L.stat('agg_pass') > passed
        # one row verified against another ring of 8 (its chunk goes to the per-proof path), one tampered proof
        vro = ring_of.copy()
        wrong = int(np.flatnonzero(ring_of < n8)[3])
        vro[wrong] = (ring_of[wrong] + 1) % n8
        bad = ref.copy()
        tampered = B - 7
        bad[tampered, 300] ^= 1
        failed = L.stat('agg_fail')
        ok, vst = verify_rings(L, P, rs, vro, wl.msg_hash, bad, rlen, vt, K)
        assert L.stat('agg_fail') > failed
        ok1, st1 = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        for r in range(len(sizes)):
            rows = np.flatnonzero(vro == r)
            if not len(rows):
                continue
            vts = L.verify_tape_len_ex(sizes[r], S, K)
            o, s = np.zeros(len(rows), np.uint8), np.zeros(len(rows), np.int32)
            pr = bad[rows].copy()
            L.verify_batch_ex(P, len(rows), wl.msg_hash[rows].copy(), wl.rings[r], sizes[r], pr, ps, rlen[rows].copy(),
                              vt[rows][:, :vts].copy(), vts, o, s, K)
            ok1[rows], st1[rows] = o, s
        assert np.array_equal(ok, ok1) and np.array_equal(vst, st1)
        assert not ok[wrong] and not ok[tampered] and ok.sum() == B - 2
    finally:
        L.set_option('lanes', cfg['lanes'])
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)
    spots = [int(np.flatnonzero(ring_of < n8)[0])] + [int(by_ring[n8 + i][0]) for i in range(len(big_sizes))]
    if L.group != 'tomEdwards256':     # oracle/cpu restates the tomEdwards256 build: the Python oracle checks war256
        for b in spots:
            pr, _ = oracle_row(po, wl, b, tape[b].tobytes())
            assert ref[b, :rlen[b]].tobytes() == flat.ser_proof(pr), b
    else:
        g.build_oracle_cpu()
        cpu = ZkaLib(g.ORACLE_CPU)
        hn, hp = cpu.params_generate(synth.params_rnd(seed))
        Pc = cpu.params_create(hn, hp, S)
        for b in spots:
            r = int(ring_of[b])
            one = _one_ring(wl, [b], r)
            cp, cl, cs = common.run_prove(cpu, Pc, one, tape[[b]][:, :L.prove_tape_len(sizes[r], S)].copy(), S)
            assert cs[0] == 0 and cp[0, :cl[0]].tobytes() == ref[b, :rlen[b]].tobytes(), b
        cpu.params_destroy(Pc)
    rs.close()
    L.params_destroy(P)


@pytest.mark.gpu
def test_rings_on_gpu_equal_the_per_ring_calls(gpu_engine):
    # 1024 rings of 8 with one signer each, plus rings of 300 (depth 9) and 2100 (depth 12: the blocked GK kernels)
    check_gpu_rings(gpu_engine.lib, 1024, (300, 2100), 512, S=80, seed=111)


@pytest.mark.gpu
def test_rings_on_gpu_war_equal_the_per_ring_calls(gpu_engine_war):
    check_gpu_rings(gpu_engine_war.lib, 96, (17, 300), 80, S=20, seed=112)
