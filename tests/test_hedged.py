"""Hedged seeds: each proof's seed derived on the device from the caller's seed, the statement and the signature
(include/zkattest.h, "Hedged seeds"), checked against its restatement in tests/hedge_rule.py, against the seeded call on
the derived seeds and against the oracle, on the host simulator (both proof groups) and on the GPU.
"""
import ctypes as C

import numpy as np
import pytest

import common
import hedge_rule as HR
from oracle import flat
from oracle import seed_tape as ST
from oracle import zkattest as OZ
from oracle.big import Tape
from oracle.curves import p256
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT


def _seeds(rows, tag):
    return np.frombuffer(synth.Drbg(rows, f'hedge-{tag}').bytes(32 * rows), np.uint8).reshape(rows, 32).copy()


def _n(N):
    return VT.ceil_log2(N)


class Setup:
    """params of one seed / sec_level and their digest under the rule"""

    def __init__(self, L, seed, S, hn=None, hp=None):
        self.L, self.S = L, S
        self.P, self.po = common.make_params(L, seed, S)
        self.hn, self.hp = self.po.NistGroup.h.to_bytes(), self.po.ProofGroup.h.to_bytes()
        if hn is not None or hp is not None:     # another pair of h points under the same library
            L.params_destroy(self.P)
            self.hn, self.hp = hn or self.hn, hp or self.hp
            self.P = L.params_create(self.hn, self.hp, S)
        self.digest = HR.params_digest(L.group, self.hn, self.hp, S)

    def close(self):
        self.L.params_destroy(self.P)


def oracle_seeds(ps, ring, msg_hash, sig, pk, which, seeds):
    rd = HR.ring_digest([bytes(e) for e in ring])
    return [HR.hedge_seed(ps.digest, rd, None if seeds is None else seeds[b].tobytes(), msg_hash[b].tobytes(),
                          sig[b].tobytes(), pk[b].tobytes(), int(which[b])) for b in range(len(which))]


def lib_seeds(L, ps, wl, seeds, N=None, ring=None):
    ring = wl.ring if ring is None else ring
    return L.hedge_seeds(ps.P, wl.B, wl.msg_hash, wl.sig, wl.pk, wl.which, ring, ring.shape[0] if N is None else N, seeds)


def run(L, fn, P, wl, seeds, S, ring=None):
    ring = wl.ring if ring is None else ring
    B, N = wl.B, ring.shape[0]
    ps = L.proof_max_len(N, S)
    proofs, plen, st = np.zeros((B, ps), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)
    getattr(L, fn)(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, ring, N, seeds, proofs, ps, plen, st)
    return proofs, plen, st


def rows_equal(a, b):
    (pa, la, sa), (pb, lb, sb) = a, b
    return (np.array_equal(la, lb) and np.array_equal(sa, sb)
            and all(pa[i, :la[i]].tobytes() == pb[i, :lb[i]].tobytes() for i in range(len(la))))


# ------------------------------------------------------------------------------------------- 1. model = library
def check_model(L, sizes, S=16, seed=201):
    ps = Setup(L, seed, S)
    for N in sizes:
        wl = synth.Workload(B=3, N=N, seed=seed + N)
        for seeds in (_seeds(3, f'm-{N}'), None):
            got = lib_seeds(L, ps, wl, seeds)
            want = oracle_seeds(ps, wl.ring, wl.msg_hash, wl.sig, wl.pk, wl.which, seeds)
            assert [got[b].tobytes() for b in range(3)] == want, (N, seeds is None)
    ps.close()


def check_model_rings(L, S=16, seed=202):
    ps = Setup(L, seed, S)
    sizes = [17, 5, 3000, 2, 256]
    ring_of = [2, 0, 4, 1, 3, 0, 2, 1]
    rw = synth.RingsWorkload(len(ring_of), sizes, ring_of, seed=seed)
    h = L.rings_create(np.array(sizes, np.uint32), rw.keys)
    for seeds in (_seeds(len(ring_of), 'mr'), None):
        got = L.hedge_seeds_rings(ps.P, h, rw.ring_of, rw.B, rw.msg_hash, rw.sig, rw.pk, rw.which, seeds)
        for b, r in enumerate(ring_of):
            want = oracle_seeds(ps, rw.rings[r], rw.msg_hash[b:b + 1], rw.sig[b:b + 1], rw.pk[b:b + 1], rw.which[b:b + 1],
                                None if seeds is None else seeds[b:b + 1])[0]
            assert got[b].tobytes() == want, (b, r, seeds is None)
    L.rings_destroy(h)
    ps.close()


def test_hedge_seeds_match_oracle_hostsim(hostsim):
    check_model(hostsim, (2, 5, 6, 17, 256, 3000))     # 3000: four leaves of 1024, padding from entry 3000 on
    check_model_rings(hostsim)


def test_hedge_seeds_match_oracle_hostsim_war(hostsim_war):
    check_model(hostsim_war, (2, 5, 3000))
    check_model_rings(hostsim_war)


def test_ring_digest_leaves():
    # 2^n <= 1024: one leaf of all 2^n entries; 3000 -> 4096 padded entries, four leaves, the last of padding only
    ring = [i * 0x1234567 + 5 for i in range(3000)]
    enc = [(v % ST.P256_P).to_bytes(32, 'big') for v in ring] + [(ring[0] % ST.P256_P).to_bytes(32, 'big')] * 1096
    leaves = [HR.sha(*enc[k:k + 1024]) for k in range(0, 4096, 1024)]
    assert HR.ring_digest(ring) == HR.sha(b'ZKAttest/hedge/ring/v1', (3000).to_bytes(4, 'little'), (12).to_bytes(4, 'little'),
                                           *leaves)
    # entries are taken mod the proof-group order
    assert HR.ring_digest([5, ST.P256_P + 7]) == HR.ring_digest([5, 7])


# ------------------------------------------------------------------------ 2. hedged = seeded on derived = oracle
def check_hedged_prove(L, N=6, S=16, seed=211, oracle=True):
    ps = Setup(L, seed, S)
    wl = synth.Workload(B=5, N=N, seed=seed)
    wl.pk[1, 40] ^= 1                         # not a point of the curve
    wl.which[2] = 1000                        # outside the ring
    wl.which[3] = (1 << _n(N)) - 1            # inside the padding
    wl.which[4] = (1 << _n(N)) - 1
    wl.pk[4, 40] ^= 1                         # two defects: the pk wins
    seeds = _seeds(5, f'p-{seed}')
    derived = lib_seeds(L, ps, wl, seeds)
    hedged = run(L, 'prove_batch_hedged', ps.P, wl, seeds, S)
    seeded = run(L, 'prove_batch_seeded', ps.P, wl, derived, S)
    assert rows_equal(hedged, seeded)
    assert list(hedged[2]) == [0, 1, 6, 6, 1]
    proofs, plen, _ = hedged
    if oracle:
        pr = OZ.prove_signature_list(ps.po, wl.msg_hash[0].tobytes(), wl.sig[0].tobytes(), wl.pk[0].tobytes(), int(wl.which[0]),
                                     wl.ring_ints(), tp := Tape(ST.prove_tape(derived[0].tobytes(), S, _n(N))))
        assert proofs[0, :plen[0]].tobytes() == flat.ser_proof(pr)
        z = sum(1 for e in pr.expProof if e.alpha is None)
        assert tp.calls == 3 + 4 * S + 40 * z + 5 * _n(N)
        tape = L.seed_tape(0, derived, N, S)            # the expansion the library itself reports
        assert tape[0, :32 * tp.calls].tobytes() == ST.prove_tape(derived[0].tobytes(), S, _n(N))[:32 * tp.calls]
        vt = L.seed_tape(1, _seeds(1, 'v'), N, S, 5)
        prf = flat.de_proof(proofs[0, :plen[0]].tobytes(), S)
        assert OZ.verify_signature_list(ps.po, wl.msg_hash[0].tobytes(), wl.ring_ints(), prf,
                                        Tape(VT.oracle_stream(vt[0].tobytes(), N, S)), 5) is True
    ps.close()


def test_hedged_equals_seeded_and_oracle_hostsim(hostsim):
    check_hedged_prove(hostsim)


def test_hedged_equals_seeded_hostsim_war(hostsim_war):
    check_hedged_prove(hostsim_war, N=5, seed=212, oracle=False)


# --------------------------------------------------------------------------------------------------- 3. binding
def test_binding(hostsim):
    L, S = hostsim, 16
    ps = Setup(L, 221, S)
    wl = synth.Workload(B=3, N=6, seed=221, distinct_signers=2)
    seeds = _seeds(3, 'bind')
    base = lib_seeds(L, ps, wl, seeds)[0].tobytes()

    def changed(mutate, setup=ps, ring=None, N=None, sd=seeds):
        w = synth.Workload.__new__(synth.Workload)
        w.B, w.msg_hash, w.sig, w.pk, w.which = 3, wl.msg_hash.copy(), wl.sig.copy(), wl.pk.copy(), wl.which.copy()
        w.ring = wl.ring.copy() if ring is None else ring
        mutate(w)
        return lib_seeds(L, setup, w, sd, N=N)[0].tobytes() != base

    def flip(arr, i):
        def m(w):
            getattr(w, arr)[0, i] ^= 1
        return m
    assert changed(flip('msg_hash', 7))
    assert changed(flip('sig', 5))                  # r
    assert changed(flip('sig', 40))                 # s
    assert not np.array_equal(wl.pk[0], wl.pk[1])
    assert changed(lambda w: w.pk.__setitem__(0, wl.pk[1]))   # another valid key
    assert changed(lambda w: w.which.__setitem__(0, wl.which[0] ^ 1))
    for j in (0, 3, 5):                             # first, middle, last ring entry
        ring = wl.ring.copy()
        ring[j, 31] ^= 1
        assert changed(lambda w: None, ring=ring), j
    # N = 5 against N = 6 with the same padded ring (the sixth entry equal to the padding e_0)
    r6 = wl.ring.copy()
    r6[5] = r6[0]
    five = lib_seeds(L, ps, _with(wl, which=1), seeds, ring=r6[:5].copy())[0].tobytes()
    six = lib_seeds(L, ps, _with(wl, which=1), seeds, ring=r6)[0].tobytes()
    assert five != six
    other = Setup(L, 222, S)
    for hn, hp in ((other.hn, None), (None, other.hp)):
        alt = Setup(L, 221, S, hn=hn, hp=hp)
        assert changed(lambda w: None, setup=alt)
        alt.close()
    other.close()
    s20 = Setup(L, 221, 20)
    assert changed(lambda w: None, setup=s20)
    s20.close()
    sd = seeds.copy()
    sd[0, 0] ^= 1
    assert changed(lambda w: None, sd=sd)
    assert changed(lambda w: None, sd=None)
    # unchanged: the row moved inside the batch, other neighbours, or proved through a ring set
    perm = [2, 0, 1]
    moved = lib_seeds(L, ps, _with(wl, perm=perm), seeds[perm].copy())
    assert moved[1].tobytes() == base
    assert not changed(lambda w: (w.msg_hash.__setitem__(1, 0), w.sig.__setitem__(2, 1), w.which.__setitem__(2, 9)))
    h = L.rings_create(np.array([4, 6], np.uint32), np.concatenate([wl.ring[:4], wl.ring]))
    via = L.hedge_seeds_rings(ps.P, h, np.array([1, 0, 1], np.uint32), 3, wl.msg_hash, wl.sig, wl.pk, wl.which, seeds)
    assert via[0].tobytes() == base
    L.rings_destroy(h)
    ps.close()


def _with(wl, which=None, perm=None):
    w = synth.Workload.__new__(synth.Workload)
    idx = list(range(wl.B)) if perm is None else perm
    w.B, w.N, w.ring = wl.B, wl.N, wl.ring
    w.msg_hash, w.sig, w.pk, w.which = (a[idx].copy() for a in (wl.msg_hash, wl.sig, wl.pk, wl.which))
    if which is not None:
        w.which[0] = which
    return w


# ----------------------------------------------------------------------------- 4. the attack, before and after
def recovered_keys(proofs, plen, msg_hash, S):
    """What an attacker who sees two proofs and the public messages computes from every repetition pair (tag 1 in one,
    tag 0 in the other): s1 = alpha - z, then s1 * R - Q of the second statement."""
    prf = [flat.de_proof(proofs[b, :plen[b]].tobytes(), S) for b in range(2)]
    n = p256.order
    out = set()
    for a, b in ((0, 1), (1, 0)):
        R = prf[b].R
        r = R.to_affine()[0] % n
        zm = OZ.truncate_to_n(int.from_bytes(msg_hash[b].tobytes(), 'big'), n)
        negQ = p256.generator().mul(p256.new_scalar((-zm * pow(r, -1, n)) % n))
        for ea in prf[a].expProof:
            if ea.alpha is None:
                continue
            for eb in prf[b].expProof:
                if eb.alpha is not None:
                    continue
                s1 = (ea.alpha.k - eb.z.k) % n
                out.add(R.mul(p256.new_scalar(s1)).add(negQ).to_bytes())
    return out


def test_reused_seed_attack_seeded_vs_hedged(hostsim):
    L, S = hostsim, 16
    ps = Setup(L, 231, S)
    wl = synth.Workload(B=2, N=5, seed=231, distinct_signers=1)
    assert np.array_equal(wl.pk[0], wl.pk[1]) and not np.array_equal(wl.msg_hash[0], wl.msg_hash[1])
    seed = _seeds(1, 'reused')
    both = np.concatenate([seed, seed])
    pk = wl.pk[0].tobytes()
    proofs, plen, st = run(L, 'prove_batch_seeded', ps.P, wl, both, S)
    assert not st.any()
    assert pk in recovered_keys(proofs, plen, wl.msg_hash, S)           # the signer is deanonymised
    proofs, plen, st = run(L, 'prove_batch_hedged', ps.P, wl, both, S)
    assert not st.any()
    assert pk not in recovered_keys(proofs, plen, wl.msg_hash, S)       # every pair gives some other point
    ps.close()


# ----------------------------------------------------------------------------------------------- 5. determinism
def test_determinism(hostsim):
    L, S, N = hostsim, 16, 6
    ps = Setup(L, 241, S)
    wl = synth.Workload(B=3, N=N, seed=241)
    a = run(L, 'prove_batch_hedged', ps.P, wl, None, S)
    b = run(L, 'prove_batch_hedged', ps.P, wl, None, S)
    assert not a[2].any() and rows_equal(a, b)
    perm = [1, 2, 0]
    c = run(L, 'prove_batch_hedged', ps.P, _with(wl, perm=perm), None, S)
    assert rows_equal(tuple(x[perm] for x in a), c)
    s1 = run(L, 'prove_batch_hedged', ps.P, wl, _seeds(3, 'd1'), S)
    s2 = run(L, 'prove_batch_hedged', ps.P, wl, _seeds(3, 'd2'), S)
    vt = L.seed_tape(1, _seeds(1, 'dv'), N, S, 5)
    for proofs, plen, st in (s1, s2):
        assert not st.any()
        prf = flat.de_proof(proofs[0, :plen[0]].tobytes(), S)
        assert OZ.verify_signature_list(ps.po, wl.msg_hash[0].tobytes(), wl.ring_ints(), prf,
                                        Tape(VT.oracle_stream(vt[0].tobytes(), N, S)), 5) is True
    assert s1[0][0, :s1[1][0]].tobytes() != s2[0][0, :s2[1][0]].tobytes()
    assert a[0][0, :a[1][0]].tobytes() != s1[0][0, :s1[1][0]].tobytes()
    ps.close()


# ------------------------------------------------------------------------------------------------- 6. ring sets
def check_rings(L, sizes, ring_of, S, seed):
    ps = Setup(L, seed, S)
    rw = synth.RingsWorkload(len(ring_of), sizes, ring_of, seed=seed)
    h = L.rings_create(np.array(sizes, np.uint32), rw.keys)
    B = rw.B
    ps_len = max(L.proof_max_len(sizes[r], S) for r in set(ring_of))
    seeds = _seeds(B, f'r-{seed}')
    proofs, plen, st = np.zeros((B, ps_len), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)
    n0 = L.launch_count()
    L.prove_batch_rings_hedged(ps.P, h, rw.ring_of, B, rw.msg_hash, rw.sig, rw.pk, rw.which, seeds, proofs, ps_len, plen, st)
    n1 = L.launch_count()
    assert not st.any()
    for r in sorted(set(ring_of)):     # each row = the one-ring hedged call on its ring (row position does not matter)
        rows = [b for b in range(B) if ring_of[b] == r]
        w = synth.Workload.__new__(synth.Workload)
        w.B, w.ring = len(rows), rw.rings[r]
        w.msg_hash, w.sig, w.pk, w.which = (a[rows].copy() for a in (rw.msg_hash, rw.sig, rw.pk, rw.which))
        one = run(L, 'prove_batch_hedged', ps.P, w, seeds[rows].copy(), S)
        for i, b in enumerate(rows):
            assert one[1][i] == plen[b] and one[0][i, :plen[b]].tobytes() == proofs[b, :plen[b]].tobytes(), (r, b)
    # one SeedHedgeTask per chunk more than the seeded call, and no digest launch (done by zka_rings_create)
    derived = L.hedge_seeds_rings(ps.P, h, rw.ring_of, B, rw.msg_hash, rw.sig, rw.pk, rw.which, seeds)
    p2, l2, s2 = np.zeros_like(proofs), np.zeros_like(plen), np.zeros_like(st)
    n2 = L.launch_count()
    L.prove_batch_rings_seeded(ps.P, h, rw.ring_of, B, rw.msg_hash, rw.sig, rw.pk, rw.which, derived, p2, ps_len, l2, s2)
    n3 = L.launch_count()
    assert rows_equal((proofs, plen, st), (p2, l2, s2))
    assert (n1 - n0) - (n3 - n2) == len(L.chunk_schedule(B, True)) - 1
    L.rings_destroy(h)
    ps.close()


def test_rings_mixed_depths_hostsim(hostsim):
    check_rings(hostsim, [5, 17, 2], [1, 0, 2, 1, 0], S=16, seed=251)


def test_rings_mixed_depths_hostsim_war(hostsim_war):
    check_rings(hostsim_war, [3, 9], [1, 0, 1], S=16, seed=252)


def check_one_ring_launches(L, wl, S, seeds, ps):
    """one SeedHedgeTask per chunk and the two ring-digest launches more than the seeded call on the derived seeds"""
    derived = lib_seeds(L, ps, wl, seeds)
    run(L, 'prove_batch_seeded', ps.P, wl, derived, S)          # warm: the Lagrange matrix of this depth is cached
    n0 = L.launch_count()
    h = run(L, 'prove_batch_hedged', ps.P, wl, seeds, S)
    n1 = L.launch_count()
    s = run(L, 'prove_batch_seeded', ps.P, wl, derived, S)
    n2 = L.launch_count()
    assert rows_equal(h, s)
    assert (n1 - n0) - (n2 - n1) == len(L.chunk_schedule(wl.B, True)) - 1 + 2


def test_one_ring_launch_count_hostsim(hostsim):
    ps = Setup(hostsim, 261, 16)
    check_one_ring_launches(hostsim, synth.Workload(B=2, N=6, seed=261), 16, _seeds(2, 'lc'), ps)
    ps.close()


# -------------------------------------------------------------------------------------------- 7. argument checks
def test_argument_checks(hostsim):
    L, S = hostsim, 16
    ps = Setup(L, 271, S)
    wl = synth.Workload(B=2, N=6, seed=271)
    P = ps.P
    pl = L.proof_max_len(6, S)
    proofs, plen, st = np.zeros((2, pl), np.uint8), np.zeros(2, np.uint32), np.zeros(2, np.int32)
    seeds = _seeds(2, 'args')
    out = np.zeros((2, 32), np.uint8)
    p = C.c_void_p
    ptr = lambda a: p(a.ctypes.data)   # noqa: E731
    lib, ctx = L.lib, L.ctx

    def prove(fn, rnd, B=2, N=6, msg=ptr(wl.msg_hash), stride=pl):
        return getattr(lib, f'zka_prove_batch_{fn}')(ctx, P, B, msg, ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), N, rnd,
                                                      ptr(proofs), stride, ptr(plen), ptr(st))

    for B, N in ((0, 6), (2, 1), (2, (1 << 20) + 1), (2, 6)):
        assert prove('hedged', ptr(seeds), B, N) == prove('seeded', ptr(seeds), B, N), (B, N)
    assert prove('hedged', ptr(seeds), msg=p(0)) == prove('seeded', ptr(seeds), msg=p(0)) == -1
    assert prove('hedged', ptr(seeds), stride=pl - 1) == prove('seeded', ptr(seeds), stride=pl - 1) == -1
    assert prove('seeded', p(0)) == -1 and prove('hedged', p(0)) == 0    # NULL seeds: the hedged calls only
    assert lib.zka_hedge_seeds(ctx, P, 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), 6, p(0), ptr(out)) == 0
    assert lib.zka_hedge_seeds(ctx, P, 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), 6, p(0), p(0)) == -1
    assert lib.zka_hedge_seeds(ctx, P, 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), 1, p(0), ptr(out)) == -1
    # ring sets: a ring index >= R is rejected before any work
    h = L.rings_create(np.array([6, 3], np.uint32), np.concatenate([wl.ring, wl.ring[:3]]))
    bad = np.array([0, 2], np.uint32)
    st[:] = 77
    n0 = L.launch_count()
    for fn in ('hedged', 'seeded'):
        assert getattr(lib, f'zka_prove_batch_rings_{fn}')(ctx, P, h, ptr(bad), 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk),
                                                            ptr(wl.which), ptr(seeds), ptr(proofs), pl, ptr(plen), ptr(st)) == -1
    assert lib.zka_prove_batch_rings_hedged(ctx, P, h, ptr(bad), 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), p(0),
                                            ptr(proofs), pl, ptr(plen), ptr(st)) == -1
    assert lib.zka_hedge_seeds_rings(ctx, P, h, ptr(bad), 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), p(0),
                                     ptr(out)) == -1
    assert L.launch_count() == n0 and (st == 77).all()
    assert lib.zka_prove_batch_rings_hedged(ctx, P, h, p(0), 2, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), p(0),
                                            ptr(proofs), pl, ptr(plen), ptr(st)) == -1
    L.rings_destroy(h)
    ps.close()


def test_engine_hedged_defaults(hostsim, monkeypatch):
    """Engine.prove_batch_hedged draws os.urandom(32 * B) by default; deterministic=True passes no seeds."""
    from zkp_ecdsa_b200 import api
    eng = api.Engine.__new__(api.Engine)
    eng.lib, eng.proof_group = hostsim, hostsim.group
    ps = Setup(hostsim, 281, 16)
    params = type('P', (), {'handle': ps.P, 'sec_level': 16})()
    wl = synth.Workload(B=2, N=5, seed=281)
    drawn = []
    real = api.os.urandom
    monkeypatch.setattr(api.os, 'urandom', lambda n: drawn.append(real(n)) or drawn[-1])
    res = eng.prove_batch_hedged(params, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring)
    assert (res.status == 0).all() and [len(b) for b in drawn] == [64]
    want = lib_seeds(hostsim, ps, wl, np.frombuffer(drawn[0], np.uint8).reshape(2, 32).copy())
    seeded = run(hostsim, 'prove_batch_seeded', ps.P, wl, want, 16)
    assert rows_equal((res.proofs, res.proof_len, res.status), seeded)
    det = eng.prove_batch_hedged(params, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, deterministic=True)
    assert len(drawn) == 1
    assert rows_equal((det.proofs, det.proof_len, det.status), run(hostsim, 'prove_batch_hedged', ps.P, wl, None, 16))
    assert np.array_equal(eng.hedge_seeds(params, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, deterministic=True),
                          lib_seeds(hostsim, ps, wl, None))
    with pytest.raises(ValueError):
        eng.prove_batch_hedged(params, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, seeds=want, deterministic=True)
    ps.close()


# ------------------------------------------------------------------------------------------------------------- GPU
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check_gpu_hedged(L, B=512, N=256, S=80, seed=291):
    import torch
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    ps = Setup(L, seed, S)
    wl = synth.Workload(B=B, N=N, seed=seed)
    seeds = _seeds(B, f'gpu-{seed}')
    derived = lib_seeds(L, ps, wl, seeds)
    assert [derived[b].tobytes() for b in (0, B - 1)] == [oracle_seeds(ps, wl.ring, wl.msg_hash, wl.sig, wl.pk, wl.which, seeds)[b]
                                                         for b in (0, B - 1)]
    ref = run(L, 'prove_batch_seeded', ps.P, wl, derived, S)
    assert not ref[2].any()
    pl = L.proof_max_len(N, S)
    cfg = L.config()
    try:
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            for chunk in (None, 128):
                if chunk:
                    L.set_option('chunk', chunk)
                    L.set_option('host_chunk', chunk)
                assert rows_equal(run(L, 'prove_batch_hedged', ps.P, wl, seeds, S), ref), ('host', lanes, chunk)
                dp = torch.zeros(B * pl, dtype=torch.uint8, device='cuda')
                dl = torch.zeros(B, dtype=torch.int32, device='cuda')
                ds = torch.zeros(B, dtype=torch.int32, device='cuda')
                dm, dsig, dpk, dw, dr, dseed = (_dev(x) for x in (wl.msg_hash, wl.sig, wl.pk, wl.which.view(np.int32), wl.ring, seeds))
                L.prove_batch_hedged(ps.P, B, dm.data_ptr(), dsig.data_ptr(), dpk.data_ptr(), dw.data_ptr(), dr.data_ptr(), N,
                                     dseed.data_ptr(), dp.data_ptr(), pl, dl.data_ptr(), ds.data_ptr())
                torch.cuda.synchronize()
                got = (dp.cpu().numpy().reshape(B, pl), dl.cpu().numpy().view(np.uint32), ds.cpu().numpy())
                assert rows_equal(got, ref), ('device', lanes, chunk)
                dout = torch.zeros(B * 32, dtype=torch.uint8, device='cuda')
                L.hedge_seeds(ps.P, B, dm.data_ptr(), dsig.data_ptr(), dpk.data_ptr(), dw.data_ptr(), dr.data_ptr(), N,
                              dseed.data_ptr(), dout.data_ptr())
                torch.cuda.synchronize()
                assert np.array_equal(dout.cpu().numpy().reshape(B, 32), derived)
                L.set_option('chunk', cfg['chunk'])
                L.set_option('host_chunk', 2048)
    finally:
        L.set_option('lanes', cfg['lanes'])
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)
    det = lib_seeds(L, ps, wl, None)
    assert rows_equal(run(L, 'prove_batch_hedged', ps.P, wl, None, S), run(L, 'prove_batch_seeded', ps.P, wl, det, S))
    check_one_ring_launches(L, wl, S, seeds, ps)
    tape = L.seed_tape(0, derived, N, S)
    proofs, plen, _ = ref
    spots = [0, B - 1]
    if L.group != 'tomEdwards256':     # oracle/cpu restates the tomEdwards256 build: the Python oracle checks war256
        for b in spots:
            pr, _ = common.oracle_proof(ps.po, wl, tape, b)
            assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), b
        ps.close()
        return
    g.build_oracle_cpu()
    cpu = ZkaLib(g.ORACLE_CPU)
    hn, hp = cpu.params_generate(synth.params_rnd(seed))
    Pc = cpu.params_create(hn, hp, S)
    sub = _with(wl, perm=spots)
    sub.B, sub.N = len(spots), N
    cp, cl, cs = common.run_prove(cpu, Pc, sub, tape[spots].copy(), S)
    assert not cs.any()
    for i, b in enumerate(spots):
        assert cp[i, :cl[i]].tobytes() == proofs[b, :plen[b]].tobytes(), b
    cpu.params_destroy(Pc)
    ps.close()


@pytest.mark.gpu
def test_hedged_on_gpu_equals_seeded(gpu_engine):
    check_gpu_hedged(gpu_engine.lib)


@pytest.mark.gpu
def test_hedged_on_gpu_war_equals_seeded(gpu_engine_war):
    check_gpu_hedged(gpu_engine_war.lib, B=256, N=17, S=16, seed=292)


MIXED_SIZES = [8, 1024, 3, 256, 17, 64, 2, 600]


@pytest.mark.gpu
def test_hedged_rings_on_gpu_equal_one_ring_calls(gpu_engine):
    rng = np.random.default_rng(293)
    check_rings(gpu_engine.lib, MIXED_SIZES, [int(v) for v in rng.integers(0, len(MIXED_SIZES), 8192)], S=80, seed=293)


@pytest.mark.gpu
def test_hedged_rings_on_gpu_war_equal_one_ring_calls(gpu_engine_war):
    rng = np.random.default_rng(294)
    check_rings(gpu_engine_war.lib, [5, 64, 17], [int(v) for v in rng.integers(0, 3, 1024)], S=16, seed=294)


@pytest.mark.gpu
def test_hedge_seeds_on_gpu_match_oracle(gpu_engine, gpu_engine_war):
    for L in (gpu_engine.lib, gpu_engine_war.lib):
        check_model(L, (2, 5, 6, 17, 256, 3000))
        check_model_rings(L)
