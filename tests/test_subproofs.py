"""Stand-alone sub-proof verifiers (SURVEY.md 8(f) row 2): zka_verify_exp_batch and zka_verify_membership_batch against the
oracle's verifyExp / verifyMembership (restating /root/reference/src/exp/exp.ts:233, src/proofGK/gk.ts:197) — the shapes
of the reference's own unit tests (test/exp/exp.test.ts: no Q, arbitrary base; test/proofGK/gk.test.ts: ring [3,5,7,11,13])."""
import numpy as np
import pytest

import common
from oracle import commit as OC
from oracle import exp as OE
from oracle import flat
from oracle import gk as OG
from oracle.big import Tape
from oracle.curves import p256, tomEdwards256 as tom
from zkp_ecdsa_b200 import synth


def _pad(rows, width=None):
    width = width or max(len(r) for r in rows)
    a = np.zeros((len(rows), max(width, 1)), np.uint8)
    for i, r in enumerate(rows):
        a[i, :len(r)] = np.frombuffer(bytes(r), np.uint8)
    return a, np.array([len(r) for r in rows], np.uint32)


def check_verify_exp(L, sec=12, K=12, with_q=False, seed=7, tampers=3):
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, sec)
    d = synth.Drbg(seed, 'subexp')
    n_ord = p256.order
    s = d.below(n_ord)
    base = p256.generator().mul(p256.new_scalar(d.below(n_ord)))
    Q = p256.generator().mul(p256.new_scalar(d.below(n_ord))) if with_q else None
    pk = base.mul(p256.new_scalar(s))
    if Q is not None:
        pk = pk.sub(Q)                       # statement: s*base - Q = pk (exp.ts:186-190)
    x, y = pk.to_affine()
    ptape = Tape(synth.random_tape(1, 32 * (3 + 4 * sec + 40 * sec + 8), seed=seed + 1)[0].tobytes())
    nist = OC.PedersenParams(p256, base, po.NistGroup.h)
    Cs = nist.commit(s, ptape)
    Cx, Cy = po.ProofGroup.commit(x, ptape), po.ProofGroup.commit(y, ptape)
    pi = OE.prove_exp(nist, po.ProofGroup, s, Cs, pk, Cx, Cy, sec, ptape, Q)
    body = b''.join(flat.ser_exp(e) for e in pi)
    cases = [bytearray(body)]
    rng = np.random.default_rng(seed)
    for _ in range(tampers):
        b = bytearray(body)
        b[int(rng.integers(200, len(b) - 40))] ^= 1 << int(rng.integers(0, 8))
        cases.append(b)
    T = len(cases)
    proofs, lens = _pad(cases)
    rep = lambda a: np.repeat(np.frombuffer(a, np.uint8)[None, :], T, axis=0).copy()   # noqa: E731
    tape = synth.random_tape(T, 96 + 32 * 25 * K, seed=seed + 2)
    idx_rng = np.random.default_rng(seed + 3)
    for i in range(sec - 2):
        tape[:, i] = idx_rng.integers(0, sec - i, size=T, dtype=np.uint8)
    tape[:, sec - 2:96] = 0
    qarr = rep(flat._pt(Q, 65)) if Q is not None else None
    ok, st = L.verify_exp_batch(P, rep(flat._pt(base, 65)), rep(flat._pt(Cs.p, 65)), rep(Cx.p.to_bytes()), rep(Cy.p.to_bytes()), qarr,
                                proofs, lens, tape, K)
    assert ok[0] == 1 and st[0] == 0
    for i in range(T):
        stream = bytes(tape[i, :sec - 2]) + bytes(tape[i, 96:])
        try:
            r = flat._Rd(bytes(cases[i]))
            reps = []
            for _k in range(sec):
                tag = r.take(1)[0]
                A, Tx, Ty = r.npt(), r.wpt(), r.wpt()
                if tag == 1:
                    reps.append(OE.ExpProof(A, Tx, Ty, r.nsc(), r.nsc(), r.wsc(), r.wsc()))
                elif tag == 0:
                    z, z2 = r.nsc(), r.nsc()
                    pa = flat._de_pa(r)
                    reps.append(OE.ExpProof(A, Tx, Ty, None, None, None, None, z, z2, pa, r.wsc(), r.wsc()))
                else:
                    raise ValueError('tag')
            if r.o != len(r.b):
                raise ValueError('trailing')
            exp = OE.verify_exp(nist, po.ProofGroup, Cs.p, Cx.p, Cy.p, reps, K, Tape(stream), Q)
        except ValueError:
            exp = 'err'
        got = 'err' if st[i] else bool(ok[i])
        assert got == exp, (i, got, int(st[i]), exp)
    L.params_destroy(P)


def check_verify_membership(L, ring_vals, index, seed=9, tampers=3):
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    ptape = Tape(synth.random_tape(1, 32 * 200, seed=seed + 1)[0].tobytes())
    com = params.commit(ring_vals[index], ptape)
    proof = OG.prove_membership(params, com, index, ring_vals, ptape)
    body = flat.ser_gk(proof)
    n = len(proof.cl)
    cases = [bytearray(body)]
    rng = np.random.default_rng(seed)
    for k in range(tampers):
        b = bytearray(body)
        if k == 0:
            b[len(b) - 1] ^= 1                        # zd
        else:
            b[int(rng.integers(1, len(b)))] ^= 1 << int(rng.integers(0, 8))
        cases.append(b)
    T = len(cases)
    proofs, lens = _pad(cases)
    N = len(ring_vals)
    ring = np.array([list(int(v % tom.order).to_bytes(32, 'big')) for v in ring_vals], np.uint8)
    tape = synth.random_tape(T, 32 * (2 * n + 1), seed=seed + 2)
    comb = np.repeat(np.frombuffer(com.p.to_bytes(), np.uint8)[None, :], T, axis=0).copy()
    ok, st = L.verify_membership_batch(P, comb, ring, proofs, lens, tape)
    assert ok[0] == 1 and st[0] == 0
    # a different commitment with the valid proof must fail
    other = params.commit(ring_vals[(index + 1) % N], ptape)
    ok2, st2 = L.verify_membership_batch(P, np.frombuffer(other.p.to_bytes(), np.uint8)[None, :].copy(), ring, proofs[:1].copy(), lens[:1].copy(),
                                         tape[:1].copy())
    assert ok2[0] == 0 and st2[0] == 0
    for i in range(T):
        try:
            r = flat._Rd(bytes(cases[i]))
            m = r.take(1)[0]
            arrs = [[r.wpt() for _ in range(m)] for _ in range(4)]
            scs = [[r.wsc() for _ in range(m)] for _ in range(3)]
            zd = r.wsc()
            if r.o != len(r.b):
                raise ValueError('trailing')
            exp = OG.verify_membership(params, com.p, ring_vals, OG.GKProof(*arrs, *scs, zd), Tape(tape[i].tobytes()))
        except ValueError:
            exp = 'err'
        got = 'err' if st[i] else bool(ok[i])
        assert got == exp, (i, got, int(st[i]), exp)
    L.params_destroy(P)


def test_verify_exp_without_q(hostsim):
    check_verify_exp(hostsim, sec=12, K=12, with_q=False)


def test_verify_exp_with_q_and_partial_sampling(hostsim):
    check_verify_exp(hostsim, sec=14, K=5, with_q=True, seed=17)


def test_verify_membership_reference_test_shape(hostsim):
    check_verify_membership(hostsim, [3, 5, 7, 11, 13], 3)          # test/proofGK/gk.test.ts:24-28


def test_verify_membership_ring_of_two(hostsim):
    check_verify_membership(hostsim, [1234567, 89], 1, seed=19, tampers=2)


@pytest.mark.gpu
def test_subproof_verifiers_on_gpu(gpu_engine):
    L = gpu_engine.lib
    check_verify_exp(L, sec=20, K=20, with_q=False, seed=27)
    check_verify_exp(L, sec=16, K=7, with_q=True, seed=28)
    check_verify_membership(L, [3, 5, 7, 11, 13], 3, seed=29)
    check_verify_membership(L, list(range(100, 100 + 37)), 20, seed=30)


def check_verify_small(L, kind, seed=31, tampers=3):
    """verifyEquality / verifyMult / verifyPointAdd alone against the oracle, valid + tampered, same randomizers."""
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    q = tom.order
    d = synth.Drbg(seed, 'sub' + kind)
    ptape = Tape(synth.random_tape(1, 32 * 400, seed=seed + 1)[0].tobytes())
    if kind == 'equality':                       # test/commit/equality.test.ts:26-31
        x = d.below(q)
        C1, C2 = params.commit(x, ptape), params.commit(x, ptape)
        pi = OC.prove_equality(params, x, C1, C2, ptape)
        pts, body, draws = [C1.p, C2.p], flat.ser_equality(pi), 2
        de = lambda r: flat._de_eq(r)                                                           # noqa: E731
        ver = lambda pr, tp: OC.verify_equality(params, C1.p, C2.p, pr, tp)                     # noqa: E731
    elif kind == 'mult':                         # test/commit/mult.test.ts
        x, y = d.below(q), d.below(q)
        z = x * y % q
        Cx, Cy, Cz = params.commit(x, ptape), params.commit(y, ptape), params.commit(z, ptape)
        pi = OC.prove_mult(params, x, y, z, Cx, Cy, Cz, ptape)
        pts, body, draws = [Cx.p, Cy.p, Cz.p], flat.ser_mult(pi), 5
        de = lambda r: flat._de_mult(r)                                                         # noqa: E731
        ver = lambda pr, tp: OC.verify_mult(params, Cx.p, Cy.p, Cz.p, pr, tp)                   # noqa: E731
    else:                                        # test/exp/pointAdd.test.ts
        Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Qp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Rp = Pp.add(Qp)
        (x1, y1), (x2, y2), (x3, y3) = Pp.to_affine(), Qp.to_affine(), Rp.to_affine()
        cs = [params.commit(v, ptape) for v in (x1, y1, x2, y2, x3, y3)]
        pi = OE.prove_point_add(params, Pp, Qp, Rp, *cs, ptape)
        pts, body, draws = [c.p for c in cs], flat.ser_point_add(pi), 24
        de = lambda r: flat._de_pa(r)                                                           # noqa: E731
        ver = lambda pr, tp: OE.verify_point_add(params, *[c.p for c in cs], pr, tp)            # noqa: E731
    cases = [bytearray(body)]
    rng = np.random.default_rng(seed)
    for k in range(tampers):
        b = bytearray(body)
        b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
        cases.append(b)
    T = len(cases)
    proofs = np.array([list(c) for c in cases], np.uint8)
    pbytes = b''.join(p.to_bytes() for p in pts)
    points = np.repeat(np.frombuffer(pbytes, np.uint8)[None, :], T, axis=0).copy()
    # one more case: a wrong statement (first input replaced by another valid commitment) with the valid proof
    other = params.commit(d.below(q), ptape).p.to_bytes()
    points = np.concatenate([points, np.frombuffer(other + pbytes[getattr(L, 'wp', 67):], np.uint8)[None, :]], axis=0)
    proofs = np.concatenate([proofs, proofs[:1]], axis=0)
    T += 1
    tape = synth.random_tape(T, 32 * draws, seed=seed + 2)
    ok, st = L.verify_sub_batch(kind, P, points, proofs, tape)
    assert ok[0] == 1 and st[0] == 0 and ok[T - 1] == 0 and st[T - 1] == 0
    for i in range(T - 1):
        try:
            r = flat._Rd(bytes(cases[i]))
            pr = de(r)
            exp = ver(pr, Tape(tape[i].tobytes()))
        except ValueError:
            exp = 'err'
        got = 'err' if st[i] else bool(ok[i])
        assert got == exp, (kind, i, got, int(st[i]), exp)
    L.params_destroy(P)


@pytest.mark.parametrize('kind', ['equality', 'mult', 'pointadd'])
def test_verify_small_subproofs(hostsim, kind):
    check_verify_small(hostsim, kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['equality', 'mult', 'pointadd'])
def test_verify_small_subproofs_on_gpu(gpu_engine, kind):
    check_verify_small(gpu_engine.lib, kind, seed=41, tampers=6)


def check_prove_exp(L, sec=10, with_q=False, seed=51, B=2):
    """zka_prove_exp_batch == oracle proveExp byte for byte (arbitrary base, optional Q), its output verifies with
    zka_verify_exp_batch, and a false statement reports "Points don't add up!"."""
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, sec)
    d = synth.Drbg(seed, 'provexp')
    n_ord, q = p256.order, tom.order
    ndraw = 3 + 4 * sec + 40 * sec
    tape = synth.random_tape(B + 1, 32 * ndraw, seed=seed + 1)
    base_b, s_b, pk_b, q_b, want = [], [], [], [], []
    for b in range(B + 1):
        s = d.below(n_ord)
        base = p256.generator().mul(p256.new_scalar(d.below(n_ord)))
        Q = p256.generator().mul(p256.new_scalar(d.below(n_ord))) if with_q else None
        pk = base.mul(p256.new_scalar(s))
        if Q is not None:
            pk = pk.sub(Q)
        if b == B:                                  # false statement: another public key
            pk = pk.add(p256.generator())
        x, y = pk.to_affine()
        tp = Tape(tape[b].tobytes())
        nist = OC.PedersenParams(p256, base, po.NistGroup.h)
        Cs = nist.commit(s, tp)                     # draw 0
        Cx, Cy = po.ProofGroup.commit(x, tp), po.ProofGroup.commit(y, tp)   # draws 1, 2
        try:
            pi = OE.prove_exp(nist, po.ProofGroup, s, Cs, pk, Cx, Cy, sec, tp, Q)
            want.append((b''.join(flat.ser_exp(e) for e in pi), nist, Cs, Cx, Cy, Q, base))
        except ValueError as e:
            assert "don't add up" in str(e)
            want.append(None)
        base_b.append(flat._pt(base, 65)); s_b.append(s.to_bytes(32, 'big')); pk_b.append(flat._pt(pk, 65))
        q_b.append(flat._pt(Q, 65) if Q is not None else bytes(65))
    arr = lambda rows: np.array([list(r) for r in rows], np.uint8)   # noqa: E731
    proofs, plen, st = L.prove_exp_batch(P, arr(base_b), arr(s_b), arr(pk_b), arr(q_b) if with_q else None, tape, sec)
    assert list(st[:B]) == [0] * B and st[B] == 4 and plen[B] == 0 and want[B] is None
    for b in range(B):
        assert proofs[b, :plen[b]].tobytes() == want[b][0], b
    # round trip through the stand-alone verifier
    K = sec
    vt = synth.random_tape(B, 96 + 32 * 25 * K, seed=seed + 2)
    rng = np.random.default_rng(seed)
    for i in range(sec - 2):
        vt[:, i] = rng.integers(0, sec - i, size=B, dtype=np.uint8)
    vt[:, sec - 2:96] = 0
    ok, vst = L.verify_exp_batch(P, arr(base_b[:B]), arr([flat._pt(w[2].p, 65) for w in want[:B]]), arr([w[3].p.to_bytes() for w in want[:B]]),
                                 arr([w[4].p.to_bytes() for w in want[:B]]), arr(q_b[:B]) if with_q else None,
                                 np.ascontiguousarray(proofs[:B]), plen[:B].copy(), vt, K)
    assert (ok == 1).all() and not vst.any()
    L.params_destroy(P)


def check_prove_membership(L, ring_vals, indices, seed=61):
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    N = len(ring_vals)
    n = len(bin(N - 1)) - 2
    B = len(indices)
    tape = synth.random_tape(B, 32 * 5 * n, seed=seed + 1)
    rs = synth.random_tape(B, 32, seed=seed + 2)
    want = []
    for b, idx in enumerate(indices):
        r = int.from_bytes(rs[b].tobytes(), 'big')
        com = OC.Commitment(OG.gk_commit(params, ring_vals[idx] % tom.order, r), tom.new_scalar(r))
        want.append((flat.ser_gk(OG.prove_membership(params, com, idx, ring_vals, Tape(tape[b].tobytes()))), com))
    ring = np.array([list(int(v % tom.order).to_bytes(32, 'big')) for v in ring_vals], np.uint8)
    idx_arr = np.array(list(indices) + [N + 5], np.uint32)          # one index outside the ring
    proofs, plen, st = L.prove_membership_batch(P, np.concatenate([rs, rs[:1]]), idx_arr, ring, np.concatenate([tape, tape[:1]]))
    assert list(st) == [0] * B + [6] and plen[B] == 0
    for b in range(B):
        assert proofs[b, :plen[b]].tobytes() == want[b][0], b
    vt = synth.random_tape(B, 32 * (2 * n + 1), seed=seed + 3)
    ok, vst = L.verify_membership_batch(P, np.array([list(w[1].p.to_bytes()) for w in want], np.uint8), ring,
                                        np.ascontiguousarray(proofs[:B]), plen[:B].copy(), vt)
    assert (ok == 1).all() and not vst.any()
    L.params_destroy(P)


def test_prove_exp_alone_without_q(hostsim):
    check_prove_exp(hostsim, sec=10, with_q=False)


def test_prove_exp_alone_with_q(hostsim):
    check_prove_exp(hostsim, sec=9, with_q=True, seed=52, B=1)


def test_prove_membership_alone(hostsim):
    check_prove_membership(hostsim, [3, 5, 7, 11, 13], [3, 0, 4])       # test/proofGK/gk.test.ts shape
    check_prove_membership(hostsim, [10 ** 30 + i for i in range(9)], [8], seed=62)


@pytest.mark.gpu
def test_subproof_provers_on_gpu(gpu_engine):
    L = gpu_engine.lib
    check_prove_exp(L, sec=20, with_q=False, seed=71, B=3)
    check_prove_exp(L, sec=12, with_q=True, seed=72, B=2)
    check_prove_membership(L, [3, 5, 7, 11, 13], [3, 0, 4], seed=73)
    check_prove_membership(L, list(range(500, 500 + 300)), [0, 299, 150, 7], seed=74)


def check_prove_small(L, kind, seed=81, B=3):
    """zka_prove_{equality,mult,pointadd}_batch == the oracle's proof bytes; outputs verify with the stand-alone verifier."""
    tom = common.pg(L)   # the library's ProofGroup (tomEdwards256 or war256)
    P, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    q = tom.order
    d = synth.Drbg(seed, 'prove' + kind)
    nd = {'equality': 3, 'mult': 7, 'pointadd': 38}[kind]
    tape = synth.random_tape(B, 32 * nd, seed=seed + 1)
    bl = synth.random_tape(B, 32 * 6, seed=seed + 2)
    rows, blind, want_pf, want_com = [], [], [], []
    i32 = lambda v: int(v).to_bytes(32, 'big')   # noqa: E731
    for b in range(B):
        r = [int.from_bytes(bl[b, 32 * i:32 * i + 32].tobytes(), 'big') for i in range(6)]
        tp = Tape(tape[b].tobytes())
        mk = lambda v, rr: OC.Commitment(params.h.dblmul(tom.new_scalar(rr), params.g, tom.new_scalar(v)), tom.new_scalar(rr))   # noqa: E731
        if kind == 'equality':
            x = d.below(q)
            C1, C2 = mk(x, r[0]), mk(x, r[1])
            pi = OC.prove_equality(params, x, C1, C2, tp)
            rows.append(i32(x) + i32(r[0]) + i32(r[1]))
            want_pf.append(flat.ser_equality(pi)); want_com.append(C1.p.to_bytes() + C2.p.to_bytes())
        elif kind == 'mult':
            x, y = d.below(q), d.below(q)
            z = x * y % q
            Cx, Cy, Cz = mk(x, r[0]), mk(y, r[1]), mk(z, r[2])
            pi = OC.prove_mult(params, x, y, z, Cx, Cy, Cz, tp)
            rows.append(i32(x) + i32(y) + i32(z) + i32(r[0]) + i32(r[1]) + i32(r[2]))
            want_pf.append(flat.ser_mult(pi)); want_com.append(Cx.p.to_bytes() + Cy.p.to_bytes() + Cz.p.to_bytes())
        else:
            Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
            Qp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
            Rp = Pp.add(Qp)
            if b == B - 1:
                Rp = Rp.add(p256.generator())          # false statement -> "Points don't add up!"
            (x1, y1), (x2, y2), (x3, y3) = Pp.to_affine(), Qp.to_affine(), Rp.to_affine()
            cs = [mk(v, rr) for v, rr in zip((x1, y1, x2, y2, x3, y3), r)]
            rows.append(flat._pt(Pp, 65) + flat._pt(Qp, 65) + flat._pt(Rp, 65))
            blind.append(b''.join(i32(v) for v in r))
            try:
                pi = OE.prove_point_add(params, Pp, Qp, Rp, *cs, tp)
                want_pf.append(flat.ser_point_add(pi)); want_com.append(b''.join(c.p.to_bytes() for c in cs))
            except ValueError:
                want_pf.append(None); want_com.append(None)
    arr = lambda rr: np.array([list(x) for x in rr], np.uint8)   # noqa: E731
    com, proofs, st = L.prove_sub_batch(kind, P, arr(rows), tape, arr(blind) if kind == 'pointadd' else None)
    good = []
    for b in range(B):
        if want_pf[b] is None:
            assert st[b] == 4 and not proofs[b].any() and not com[b].any()
        else:
            assert st[b] == 0 and proofs[b].tobytes() == want_pf[b] and com[b].tobytes() == want_com[b], (kind, b)
            good.append(b)
    vdraws = {'equality': 2, 'mult': 5, 'pointadd': 24}[kind]
    vt = synth.random_tape(len(good), 32 * vdraws, seed=seed + 3)
    ok, vst = L.verify_sub_batch(kind, P, np.ascontiguousarray(com[good]), np.ascontiguousarray(proofs[good]), vt)
    assert (ok == 1).all() and not vst.any()
    L.params_destroy(P)


@pytest.mark.parametrize('kind', ['equality', 'mult', 'pointadd'])
def test_prove_small_subproofs(hostsim, kind):
    check_prove_small(hostsim, kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['equality', 'mult', 'pointadd'])
def test_prove_small_subproofs_on_gpu(gpu_engine, kind):
    check_prove_small(gpu_engine.lib, kind, seed=91, B=5)


@pytest.mark.gpu
def test_subproof_chunk_loops_on_gpu(gpu_engine):
    """The stand-alone paths cut a batch into chunks of 16384 rows (proveEquality, proveMult), 8192 (provePointAdd,
    proveMembership, the small verifiers) or 4096 (verifyMembership).  One row past a chunk, every output row of a batch
    of one repeated input row equals the output of a one-row call."""
    L = gpu_engine.lib
    tom = common.pg(L)
    q = tom.order
    P, po = common.make_params(L, 95, 8)
    d = synth.Drbg(95, 'chunks')
    i32 = lambda v: int(v).to_bytes(32, 'big')                               # noqa: E731
    row = lambda b: np.frombuffer(b, np.uint8)[None, :].copy()                # noqa: E731
    rep = lambda a, k: np.ascontiguousarray(np.repeat(a, k, axis=0))          # noqa: E731

    def same(call, n):
        """call(k) runs k copies of the input row; returns the outputs of the one-row call"""
        one, many = call(1), call(n)
        for a, b in zip(one, many):
            assert b.shape[0] == n and (b == a[:1]).all()
        return one

    bl = [d.below(q) for _ in range(6)]
    x, y = d.below(q), d.below(q)
    Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
    Qp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
    inputs = {'equality': (row(i32(x) + i32(bl[0]) + i32(bl[1])), None, 3, 2, 16385),
              'mult': (row(i32(x) + i32(y) + i32(x * y % q) + b''.join(i32(v) for v in bl[:3])), None, 7, 5, 16385),
              'pointadd': (row(flat._pt(Pp, 65) + flat._pt(Qp, 65) + flat._pt(Pp.add(Qp), 65)), row(b''.join(i32(v) for v in bl)),
                           38, 24, 8193)}
    for kind, (ins, blind, pdraws, vdraws, n) in inputs.items():
        tape = synth.random_tape(1, 32 * pdraws, seed=96)
        com, proofs, st = same(lambda k: L.prove_sub_batch(kind, P, rep(ins, k), rep(tape, k), None if blind is None else rep(blind, k)), n)
        assert st[0] == 0, kind
        vt = synth.random_tape(1, 32 * vdraws, seed=97)
        ok, vst = same(lambda k: L.verify_sub_batch(kind, P, rep(com, k), rep(proofs, k), rep(vt, k)), 8193)
        assert ok[0] == 1 and vst[0] == 0, kind

    ring_vals = [3, 5, 7, 11, 13]
    ring = np.array([list(i32(v % q)) for v in ring_vals], np.uint8)
    rs = synth.random_tape(1, 32, seed=98)
    idx = np.array([3], np.uint32)
    tape = synth.random_tape(1, 32 * 5 * 3, seed=99)
    proofs, plen, st = same(lambda k: L.prove_membership_batch(P, rep(rs, k), rep(idx, k), ring, rep(tape, k)), 8193)
    assert st[0] == 0
    com = row(OG.gk_commit(po.ProofGroup, ring_vals[3] % q, int.from_bytes(rs[0].tobytes(), 'big')).to_bytes())
    vt = synth.random_tape(1, 32 * (2 * 3 + 1), seed=100)
    ok, vst = same(lambda k: L.verify_membership_batch(P, rep(com, k), ring, rep(proofs, k), rep(plen, k), rep(vt, k)), 4097)
    assert ok[0] == 1 and vst[0] == 0
    L.params_destroy(P)
