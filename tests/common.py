"""Shared parity checks: any library object with the capi.ZkaLib interface is compared with the oracle."""
import hashlib
import os

import numpy as np

from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from oracle.curves import p256, tomEdwards256 as tom
from zkp_ecdsa_b200 import synth


def pg(L):
    """oracle group object of the library's ProofGroup ('tomEdwards256' unless the library says otherwise)"""
    from oracle.curves import war256
    g = {'tomEdwards256': tom, 'war256': war256}[getattr(L, 'group', 'tomEdwards256')]
    flat.set_proof_group(g)
    return g


def be(vals, nb):
    return np.array([list(int(v).to_bytes(nb, 'big')) for v in vals], dtype=np.uint8)


def check_field_ops(L, seed=0, count=24):
    d = synth.Drbg(seed, 'field')
    g = pg(L)
    for field, (mod, nb) in enumerate([(p256.p, 32), (p256.order, 32), (g.p, g.size_field_bytes())]):
        va = [int.from_bytes(d.bytes(40), 'big') % mod for _ in range(count)] + [0, 1, mod - 1, mod - 1]
        vb = [int.from_bytes(d.bytes(40), 'big') % mod for _ in range(count)] + [mod - 1, 0, mod - 1, 1]
        a, b = be(va, nb), be(vb, nb)
        inv = lambda x, y: pow(x, -1, mod) if x else 0  # noqa: E731
        fns = [lambda x, y: x * y % mod, lambda x, y: (x + y) % mod, lambda x, y: (x - y) % mod, inv, inv]
        for op, fn in enumerate(fns):
            out = L.field_op_batch(field, op, a, b)
            for i in range(len(va)):
                assert int.from_bytes(out[i].tobytes(), 'big') == fn(va[i], vb[i]), (field, op, i)


def check_hash(L, seed=0):
    d = synth.Drbg(seed, 'hash')
    lens = np.array([0, 1, 55, 56, 63, 64, 65, 268, 603, 1000], dtype=np.uint32)
    msgs = np.frombuffer(d.bytes(len(lens) * 1000), np.uint8).reshape(len(lens), 1000).copy()
    out = L.hash80_batch(msgs, lens)
    for i, ln in enumerate(lens):
        assert out[i].tobytes() == hashlib.sha256(msgs[i, :ln].tobytes()).digest()[:10], i


def check_p256_mul(L, seed=0, count=6):
    d = synth.Drbg(seed, 'p256mul')
    ks = [d.below(p256.order) for _ in range(count)] + [0, 1, p256.order - 1, 16, 0xf0]
    k = be(ks, 32)
    G = p256.generator()

    def enc(pt):
        e = pt.to_bytes()
        return bytes(65) if len(e) == 1 else e
    out = L.p256_mul_batch(None, k)
    for i, v in enumerate(ks):
        assert out[i].tobytes() == enc(G.mul(p256.new_scalar(v))), i
    bases = [G.mul(p256.new_scalar(d.below(p256.order))) for _ in ks]
    out = L.p256_mul_batch(np.array([list(b.to_bytes()) for b in bases], dtype=np.uint8), k)
    for i, v in enumerate(ks):
        assert out[i].tobytes() == enc(bases[i].mul(p256.new_scalar(v))), i


def small_x_point(g, start=1):
    """(x, y) on the Weierstrass group g with the smallest x >= start, by trial (p = 3 mod 4: y = r^((p+1)/4))."""
    p = g.p
    assert p % 4 == 3
    x = start
    while True:
        r = (x * x * x + g.a * x + g.b) % p
        y = pow(r, (p + 1) // 4, p)
        if y * y % p == r:
            return x, y
        x += 1


def noncanonical_enc(g, x, y):
    """SEC1 encoding of (x, y) with the x coordinate written as x + p: still on the curve mod p.  weier.ts:74-89 has
    no range check, so the reference accepts it as the point (x, y); edwards.ts:70-86 rejects it."""
    cs = g.size_field_bytes()
    return b'\x04' + (x + g.p).to_bytes(cs, 'big') + y.to_bytes(cs, 'big')


def noncanonical_tampers(good):
    """(kind, proof) pairs: a valid proof with one point replaced by a non-canonical encoding of another on-curve
    point — the P-256 `A` of the first repetition, and the proof-group keyXcom."""
    g = flat.PROOF_GROUP
    out = []
    for kind, grp, off in (('p256 A', p256, flat.HEAD_LEN + 1), ('proof group keyXcom', g, 2 * flat.NP)):
        x, y = small_x_point(p256) if grp is p256 else grp.gen
        enc = noncanonical_enc(grp, x, y)
        p = good.copy()
        p[off:off + len(enc)] = np.frombuffer(enc, np.uint8)
        out.append((kind, p))
    return out


def check_noncanonical_p256(L):
    """A P-256 point given with x + p (p256_mul_batch base, keyToInt) equals the point (x, y), as in the reference."""
    x, y = small_x_point(p256)
    enc = noncanonical_enc(p256, x, y)
    pt = p256.deserialize_point(enc)
    ks = [1, 2, 0xf0, p256.order - 1]
    out = L.p256_mul_batch(np.array([list(enc)] * len(ks), np.uint8), be(ks, 32))
    for i, k in enumerate(ks):
        assert out[i].tobytes() == pt.mul(p256.new_scalar(k)).to_bytes(), i
    xs, st = L.key_to_int(np.array([list(enc)], np.uint8))
    assert st[0] == 0 and int.from_bytes(xs[0].tobytes(), 'big') == OZ.key_to_int(enc) == x


def make_params(L, seed=0, sec_level=80):
    rnd = synth.params_rnd(seed)
    hn, hp = L.params_generate(rnd)
    po = OZ.generate_params_list(Tape(rnd), sec_level, pg(L))
    assert hn == po.NistGroup.h.to_bytes() and hp == po.ProofGroup.h.to_bytes()
    return L.params_create(hn, hp, sec_level), po


def check_tom_commit(L, P, po, seed=0, count=6):
    d = synth.Drbg(seed, 'commit')
    tom = pg(L)
    q = tom.order
    vs = [d.below(q) for _ in range(count)] + [0, 1, q - 1, 0]
    rs = [d.below(q) for _ in range(count)] + [0, q - 1, 1, 5]
    out = L.tom_commit_batch(P, be(vs, 32), be(rs, 32))
    for i in range(len(vs)):
        e = po.ProofGroup.h.dblmul(tom.new_scalar(rs[i]), po.ProofGroup.g, tom.new_scalar(vs[i])).to_bytes()
        if len(e) == 1:      # Weierstrass identity ([0x00], weier.ts:244-247): a zero-filled slot in the flat layout
            e = bytes(getattr(L, 'wp', 67))
        assert out[i].tobytes() == e, i


def run_prove(L, P, wl, tape, sec_level=80):
    B, N = wl.B, wl.N
    ps = L.proof_max_len(N, sec_level)
    proofs = np.zeros((B, ps), np.uint8)
    plen = np.zeros(B, np.uint32)
    status = np.zeros(B, np.int32)
    L.prove_batch(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, tape, tape.shape[1], proofs, ps, plen, status)
    return proofs, plen, status


def oracle_proof(po, wl, tape, b):
    tp = Tape(tape[b].tobytes())
    pr = OZ.prove_signature_list(po, wl.msg_hash[b].tobytes(), wl.sig[b].tobytes(), wl.pk[b].tobytes(),
                                 int(wl.which[b]), wl.ring_ints(), tp)
    return pr, tp


def check_prove_parity(L, B=2, N=6, seed=3, sec_level=80, make_tape=synth.random_tape):
    """make_tape(rows, stride, seed): synth.random_tape, or synth.edge_tape (edge scalars in every draw)."""
    P, po = make_params(L, seed, sec_level)
    wl = synth.Workload(B=B, N=N, seed=seed)
    tape = make_tape(B, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = run_prove(L, P, wl, tape, sec_level)
    assert (status == 0).all(), status
    n = max(1, (N - 1).bit_length())
    for b in range(B):
        pr, tp = oracle_proof(po, wl, tape, b)
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), f'proof {b} differs'
        z = sum(1 for e in pr.expProof if e.alpha is None)
        assert tp.calls == 3 + 4 * sec_level + 40 * z + 5 * n      # SURVEY.md 3.1 draw-count contract
        assert plen[b] == flat.proof_len(z, n, sec_level)
    L.params_destroy(P)
    return proofs, plen


def check_prove_few_keys(L, B=10, N=5, signers=1, seed=41, sec_level=16, spots=(0, 3, 9)):
    """Few distinct signers in a larger batch: the per-key tables of the prover get wider windows (chosen on the device
    from the number of distinct keys, key_window_bits in zk_ops.cuh); the bytes stay the oracle's."""
    P, po = make_params(L, seed, sec_level)
    wl = synth.Workload(B=B, N=N, seed=seed, distinct_signers=signers)
    tape = synth.random_tape(B, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = run_prove(L, P, wl, tape, sec_level)
    assert (status == 0).all(), status
    for b in spots:
        pr, _ = oracle_proof(po, wl, tape, b)
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), f'proof {b} differs'
    L.params_destroy(P)


# ------------------------------------------------------------------------------------- verify
def run_verify(L, P, msg_hash, ring, proofs, plen, vtape):
    B = msg_hash.shape[0]
    ok = np.zeros(B, np.uint8)
    st = np.zeros(B, np.int32)
    L.verify_batch(P, B, msg_hash, ring, ring.shape[0], proofs, proofs.shape[1], plen, vtape, vtape.shape[1], ok, st)
    return ok, st


def oracle_verdict(po, msg, ring_ints, proof_bytes, vtape_row, N, sec_level=80):
    """'err' (the reference would throw), True or False — with the SAME randomness as the GPU."""
    from zkp_ecdsa_b200 import verify_tape as VT
    try:
        prf = flat.de_proof(proof_bytes, sec_level)
        return OZ.verify_signature_list(po, msg, ring_ints, prf, Tape(VT.oracle_stream(vtape_row, N, sec_level)))
    except ValueError:
        return 'err'


def check_verify_parity(L, N=6, seed=3, tampers=24, sec_level=80, make_tape=synth.random_tape, make_vtape=None):
    """Valid proofs verify; tampered inputs give the oracle's decision (throw / false / true).  make_vtape(rows,
    stride, ring_size, sec_level, seed): verify_tape.random_verify_tape (default) or edge_verify_tape."""
    from zkp_ecdsa_b200 import verify_tape as VT
    make_vtape = make_vtape or VT.random_verify_tape
    P, po = make_params(L, seed, sec_level)
    wl = synth.Workload(B=2, N=N, seed=seed)
    tape = make_tape(2, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = run_prove(L, P, wl, tape, sec_level)
    assert (status == 0).all()
    vts = L.verify_tape_len(N, sec_level)
    vt = make_vtape(2, vts, N, sec_level, seed=seed + 7)
    ok, st = run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
    assert list(ok) == [1, 1] and list(st) == [0, 0]
    ring_ints = wl.ring_ints()
    for b in range(2):
        assert oracle_verdict(po, wl.msg_hash[b].tobytes(), ring_ints, proofs[b, :plen[b]].tobytes(),
                              vt[b].tobytes(), N, sec_level) is True
    # tampering: proofs / message / ring, decisions compared with the oracle on identical randomness
    good = proofs[0, :plen[0]].copy()
    ln = len(good)
    rng = np.random.default_rng(seed)
    cases = []
    for k in range(tampers):
        p, msg, ring = good.copy(), wl.msg_hash[0].copy(), wl.ring.copy()
        kind = k % 8
        if kind < 3:
            p[int(rng.integers(0, ln))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 3:
            p = p[:ln - 1 - int(rng.integers(0, 40))]                 # truncated
        elif kind == 4:
            p[ln - 1 - getattr(L, 'ws', 33) * int(rng.integers(0, 5))] ^= 1   # a GK response scalar
        elif kind == 5:
            msg[int(rng.integers(0, 32))] ^= 1
        elif kind == 6:
            ring[int(wl.which[0]), 31] ^= 1
        else:
            p[int(rng.integers(264, ln - 1200))] ^= 1
        cases.append((p, msg, ring))
    # non-canonical coordinates: a Weierstrass point parses (the proof is then false), a tomEdwards256 one throws
    noncanon = noncanonical_tampers(good)
    for _, p in noncanon:
        cases.append((p, wl.msg_hash[0].copy(), wl.ring.copy()))
    T = len(cases)
    vt2 = make_vtape(T, vts, N, sec_level, seed=seed + 9)
    agree = 0
    for k, (p, msg, ring) in enumerate(cases):
        arr = np.zeros((1, max(len(p), 1)), np.uint8)
        arr[0, :len(p)] = p
        ok, st = run_verify(L, P, msg.reshape(1, 32).copy(), ring, arr, np.array([len(p)], np.uint32), vt2[k:k + 1].copy())
        got = 'err' if st[0] else bool(ok[0])
        exp = oracle_verdict(po, msg.tobytes(), [int.from_bytes(ring[i].tobytes(), 'big') for i in range(N)],
                             p.tobytes(), vt2[k].tobytes(), N, sec_level)
        kind = noncanon[k - tampers][0] if k >= tampers else k % 8
        if k >= tampers and kind != 'p256 A':   # the encoding itself decides: throw on tomEdwards256, parse on war256
            assert exp == ('err' if flat.PROOF_GROUP is tom else False), (kind, exp)
        assert got == exp, (k, kind, got, int(st[0]), exp)
        agree += 1
    L.params_destroy(P)
    return agree


def check_verify_samples(L, K, N=5, seed=5, sec_level=80, B=2, tampers=4, oracle='python', make_tape=synth.random_tape,
                         make_vtape=None):
    """zka_verify_batch_ex with `K` sampled repetitions (verifyExp's secparam, exp.ts:233-262) against the oracle's
    verdicts on valid and tampered proofs under identical randomness.  oracle = 'python' or a ZkaLib of oracle/cpu."""
    from zkp_ecdsa_b200 import verify_tape as VT
    make_vtape = make_vtape or VT.random_verify_tape
    P, po = make_params(L, seed, sec_level)
    wl = synth.Workload(B=B, N=N, seed=seed)
    tape = make_tape(B, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = run_prove(L, P, wl, tape, sec_level)
    assert (status == 0).all()
    vts = L.verify_tape_len_ex(N, sec_level, K)
    assert vts == VT.verify_tape_len(N, K)
    rng = np.random.default_rng(seed)
    cases = [(proofs[b, :plen[b]].copy(), wl.msg_hash[b].copy()) for b in range(B)]
    good = proofs[0, :plen[0]]
    for k in range(tampers):
        p, msg = good.copy(), wl.msg_hash[0].copy()
        if k % 2 == 0:
            p[int(rng.integers(264, len(p) - 1200))] ^= 1 << int(rng.integers(0, 8))
        else:
            msg[int(rng.integers(0, 32))] ^= 1
        cases.append((p, msg))
    T = len(cases)
    vt = make_vtape(T, vts, N, sec_level, seed=seed + 9)
    ps = L.proof_max_len(N, sec_level)
    arr = np.zeros((T, ps), np.uint8)
    lens = np.zeros(T, np.uint32)
    msgs = np.zeros((T, 32), np.uint8)
    for i, (p, m) in enumerate(cases):
        arr[i, :len(p)] = p
        lens[i] = len(p)
        msgs[i] = m
    ok = np.zeros(T, np.uint8)
    st = np.zeros(T, np.int32)
    L.verify_batch_ex(P, T, msgs, wl.ring, N, arr, ps, lens, vt, vts, ok, st, K)
    assert list(ok[:B]) == [1] * B and not st[:B].any(), (ok[:B], st[:B])
    if oracle == 'python':
        ring_ints = wl.ring_ints()
        for i, (p, m) in enumerate(cases):
            try:
                prf = flat.de_proof(p.tobytes(), sec_level)
                exp = OZ.verify_signature_list(po, m.tobytes(), ring_ints, prf, Tape(VT.oracle_stream(vt[i].tobytes(), N, sec_level)), K)
            except ValueError:
                exp = 'err'
            got = 'err' if st[i] else bool(ok[i])
            assert got == exp, (K, i, got, int(st[i]), exp)
    else:
        hn, hp = oracle.params_generate(synth.params_rnd(seed))
        Pc = oracle.params_create(hn, hp, sec_level)
        ok2 = np.zeros(T, np.uint8)
        st2 = np.zeros(T, np.int32)
        oracle.verify_batch_ex(Pc, T, msgs, wl.ring, N, arr, ps, lens, vt, vts, ok2, st2, K)
        assert (ok == ok2).all() and ((st != 0) == (st2 != 0)).all(), (K, ok, ok2, st, st2)
        oracle.params_destroy(Pc)
    L.params_destroy(P)
