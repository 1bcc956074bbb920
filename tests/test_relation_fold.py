"""Every point and response scalar of an EqualityProof, a MultProof and a PointAddProof enters a relation of the verifier.

Each case replaces ONE statement point or proof point by another valid point, or ONE response scalar by another in-range
value, so the bytes still deserialise and the verdict comes from the relations alone.  The stand-alone verifiers
(zka_verify_{equality,mult,pointadd}_batch) and the batched verifier (zka_verify_batch_ex, every repetition sampled, the
substitutions inside one 0-bit repetition's PointAddProof and its r1, r2) are checked against the oracle's verdicts
under the same randomizers; the oracle rejects every substituted case."""
import numpy as np
import pytest

import common
from oracle import commit as OC
from oracle import exp as OE
from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from oracle.curves import p256
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT

KINDS = ('equality', 'mult', 'pointadd')


def _layout(kind, wp, ws):
    """byte offsets of the (points, response scalars) of a proof body"""
    def eq(o):
        return [o, o + wp], [o + 2 * wp + i * ws for i in range(3)]

    def mult(o):
        return [o + i * wp for i in range(6)], [o + 6 * wp + i * ws for i in range(7)]

    if kind == 'equality':
        return eq(0)
    if kind == 'mult':
        return mult(0)
    mlen, elen = 6 * wp + 7 * ws, 2 * wp + 3 * ws
    pts, scs = [i * wp for i in range(4)], []           # C8 C10 C11 C13
    for o in [4 * wp + m * mlen for m in range(4)]:
        p, s = mult(o)
        pts, scs = pts + p, scs + s
    for o in [4 * wp + 4 * mlen + e * elen for e in range(2)]:
        p, s = eq(o)
        pts, scs = pts + p, scs + s
    return pts, scs


def _substituted(buf, base, pts, scs, other, d, q, ws):
    """copies of buf, each with one point (at base + o) replaced by `other` or one scalar replaced by another value < q"""
    out = []
    for o in pts:
        b = bytearray(buf)
        b[base + o:base + o + len(other)] = other
        out.append(bytes(b))
    for o in scs:
        b = bytearray(buf)
        v = (int.from_bytes(buf[base + o:base + o + ws], 'big') + 1 + d.below(q - 1)) % q
        b[base + o:base + o + ws] = v.to_bytes(ws, 'big')
        out.append(bytes(b))
    return out


def check_standalone(L, kind, seed=201):
    tom = common.pg(L)
    wp, ws = getattr(L, 'wp', 67), getattr(L, 'ws', 33)
    P, po = common.make_params(L, seed, 8)
    params, q = po.ProofGroup, tom.order
    d = synth.Drbg(seed, 'fold' + kind)
    ptape = Tape(synth.random_tape(1, 32 * 400, seed=seed + 1)[0].tobytes())
    if kind == 'equality':
        x = d.below(q)
        cs = [params.commit(x, ptape) for _ in range(2)]
        body = flat.ser_equality(OC.prove_equality(params, x, *cs, ptape))
    elif kind == 'mult':
        x, y = d.below(q), d.below(q)
        cs = [params.commit(v, ptape) for v in (x, y, x * y % q)]
        body = flat.ser_mult(OC.prove_mult(params, x, y, x * y % q, *cs, ptape))
    else:
        Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Qp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Rp = Pp.add(Qp)
        (x1, y1), (x2, y2), (x3, y3) = Pp.to_affine(), Qp.to_affine(), Rp.to_affine()
        cs = [params.commit(v, ptape) for v in (x1, y1, x2, y2, x3, y3)]
        body = flat.ser_point_add(OE.prove_point_add(params, Pp, Qp, Rp, *cs, ptape))
    stmt = [c.p for c in cs]
    other = params.commit(d.below(q), ptape).p
    ob = other.to_bytes()
    cases = [(stmt, body)]
    cases += [(stmt[:i] + [other] + stmt[i + 1:], body) for i in range(len(stmt))]
    cases += [(stmt, b) for b in _substituted(body, 0, *_layout(kind, wp, ws), ob, d, q, ws)]
    T = len(cases)
    points = np.array([list(b''.join(p.to_bytes() for p in s)) for s, _ in cases], np.uint8)
    proofs = np.array([list(b) for _, b in cases], np.uint8)
    draws = {'equality': 2, 'mult': 5, 'pointadd': 24}[kind]
    tape = np.repeat(synth.random_tape(1, 32 * draws, seed=seed + 2), T, axis=0)
    ok, st = L.verify_sub_batch(kind, P, points, proofs, tape)
    de = {'equality': flat._de_eq, 'mult': flat._de_mult, 'pointadd': flat._de_pa}[kind]
    ver = {'equality': OC.verify_equality, 'mult': OC.verify_mult, 'pointadd': OE.verify_point_add}[kind]
    for i, (s, b) in enumerate(cases):
        try:
            exp = ver(params, *s, de(flat._Rd(b)), Tape(tape[i].tobytes()))
        except ValueError:
            exp = 'err'
        assert exp is (i == 0), (kind, i, exp)
        got = 'err' if st[i] else bool(ok[i])
        assert got == exp, (kind, i, got, int(st[i]), exp)
    L.params_destroy(P)
    return T


def check_batched(L, seed=211, sec_level=6, N=4):
    tom = common.pg(L)
    wp, ws = getattr(L, 'wp', 67), getattr(L, 'ws', 33)
    P, po = common.make_params(L, seed, sec_level)
    wl = synth.Workload(B=1, N=N, seed=seed)
    tape = synth.random_tape(1, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = common.run_prove(L, P, wl, tape, sec_level)
    assert status[0] == 0
    good = proofs[0, :plen[0]].tobytes()
    rep_head, pa_len = 1 + 65 + 2 * wp, 4 * wp + 4 * (6 * wp + 7 * ws) + 2 * (2 * wp + 3 * ws)
    off = 2 * 65 + 2 * wp
    for _ in range(sec_level):                     # first 0-bit repetition
        if good[off] == 0:
            break
        off += rep_head + 2 * 32 + 2 * ws
    assert good[off] == 0, 'no 0-bit repetition'
    pts, scs = _layout('pointadd', wp, ws)
    d = synth.Drbg(seed, 'foldbatch')
    other = po.ProofGroup.commit(d.below(tom.order), Tape(synth.random_tape(1, 32, seed=seed + 1)[0].tobytes())).p.to_bytes()
    cases = [good] + _substituted(good, off + rep_head + 2 * 32, pts, scs + [pa_len, pa_len + ws], other, d, tom.order, ws)
    T, ps = len(cases), proofs.shape[1]
    arr = np.zeros((T, ps), np.uint8)
    for i, p in enumerate(cases):
        arr[i, :len(p)] = np.frombuffer(p, np.uint8)
    lens = np.full(T, len(good), np.uint32)
    msgs = np.repeat(wl.msg_hash[:1], T, axis=0)
    vts = L.verify_tape_len_ex(N, sec_level, sec_level)
    vt = np.repeat(VT.random_verify_tape(1, vts, N, sec_level, seed=seed + 9), T, axis=0)
    ok = np.zeros(T, np.uint8)
    st = np.zeros(T, np.int32)
    L.verify_batch_ex(P, T, msgs, wl.ring, N, arr, ps, lens, vt, vts, ok, st, sec_level)
    ring_ints = wl.ring_ints()
    for i, p in enumerate(cases):
        try:
            exp = OZ.verify_signature_list(po, wl.msg_hash[0].tobytes(), ring_ints, flat.de_proof(p, sec_level),
                                           Tape(VT.oracle_stream(vt[i].tobytes(), N, sec_level)), sec_level)
        except ValueError:
            exp = 'err'
        assert exp is (i == 0), (i, exp)
        got = 'err' if st[i] else bool(ok[i])
        assert got == exp, (i, got, int(st[i]), exp)
    L.params_destroy(P)
    return T


@pytest.mark.parametrize('kind', KINDS)
def test_standalone_relations(hostsim, kind):
    check_standalone(hostsim, kind)


@pytest.mark.parametrize('kind', KINDS)
def test_standalone_relations_war256(hostsim_war, kind):
    check_standalone(hostsim_war, kind, seed=202)


def test_batched_relations(hostsim):
    check_batched(hostsim)


def test_batched_relations_war256(hostsim_war):
    check_batched(hostsim_war, seed=212)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_standalone_relations_on_gpu(gpu_engine, gpu_engine_war, kind):
    check_standalone(gpu_engine.lib, kind, seed=203)
    check_standalone(gpu_engine_war.lib, kind, seed=204)


@pytest.mark.gpu
def test_batched_relations_on_gpu(gpu_engine, gpu_engine_war):
    check_batched(gpu_engine.lib, seed=213)
    check_batched(gpu_engine_war.lib, seed=214)
