"""Edges of the prover steps shared by the batched and stand-alone paths, against the oracle.

* proveEquality / proveMult alone: statement scalars given as v + q stand for v (newScalar reduces them); a draw of q or
  2^256 - 1 is a tape-range error that zeroes the row, draws 0, 1 and q - 1 give the oracle's bytes.
* The P-256 point decoder at every prover site that reads a point (pk, the proveExp base and Q, the provePointAdd P, Q and
  R) and at the sub-operations (keyToInt, the base of p256_mul_batch): canonical and x + p encodings stand for the point;
  65 zero bytes, a tag other than 0x04 and a point off the curve give each site's status."""
import numpy as np
import pytest

import common
from oracle import commit as OC
from oracle import exp as OE
from oracle import flat
from oracle.curves import p256
from oracle.big import Tape
from zkp_ecdsa_b200 import synth

INVALID_PK, TAPE_RANGE = 1, 5
BAD = ('zeros', 'tag00', 'tag02', 'y+1')
LABELS = ('canonical', 'x+p') + BAD


def i32(v):
    return int(v).to_bytes(32, 'big')


def arr(rows):
    return np.array([list(r) for r in rows], np.uint8)


# ------------------------------------------------------------------------------ proveEquality / proveMult alone
def sub_oracle(L, po, kind, vals, rs, tape_row):
    """the oracle's (proof, commitments) of proveEquality (vals = x) / proveMult (vals = x y z) under blinders rs"""
    g, params = common.pg(L), po.ProofGroup
    cs = [OC.Commitment(params.h.dblmul(g.new_scalar(r), params.g, g.new_scalar(v)), g.new_scalar(r))
          for v, r in zip(vals * 2 if kind == 'equality' else vals, rs)]
    tp = Tape(bytes(tape_row))
    if kind == 'equality':
        body = flat.ser_equality(OC.prove_equality(params, vals[0], *cs, tp))
    else:
        body = flat.ser_mult(OC.prove_mult(params, *vals, *cs, tp))
    return body, b''.join(c.p.to_bytes() for c in cs)


def sub_statement(L, kind, d):
    """canonical statement values and blinders, each below 2^256 - q so that v + q still fits 32 bytes"""
    q = common.pg(L).order
    small = lambda: d.below(q) % ((1 << 256) - q)   # noqa: E731
    if kind == 'equality':
        return [small()], [small(), small()]
    x, y = d.below(q) >> 145, d.below(q) >> 145
    return [x, y, x * y % q], [small(), small(), small()]


def sub_row(kind, vals, rs, plus):
    """the input row (x r1 r2 / x y z rx ry rz); the scalars at the indices in `plus` are written as v + q"""
    return [v + plus_q for v, plus_q in zip(vals + rs, plus)]


def check_sub_statement_scalars(L, kind, seed):
    q = common.pg(L).order
    P, po = common.make_params(L, seed, 8)
    d = synth.Drbg(seed, 'sub-statement-' + kind)
    vals, rs = sub_statement(L, kind, d)
    nd, ns = (3, 3) if kind == 'equality' else (7, 6)
    tape = synth.random_tape(1, 32 * nd, seed=seed + 1)
    want = sub_oracle(L, po, kind, vals, rs, tape[0])
    # all canonical, all v + q, then each scalar alone as v + q
    plus = [[0] * ns, [q] * ns] + [[q if j == i else 0 for j in range(ns)] for i in range(ns)]
    rows = [b''.join(i32(v) for v in sub_row(kind, vals, rs, pl)) for pl in plus]
    com, proofs, st = L.prove_sub_batch(kind, P, arr(rows), np.repeat(tape, len(rows), axis=0))
    for i in range(len(rows)):
        assert st[i] == 0 and proofs[i].tobytes() == want[0] and com[i].tobytes() == want[1], (kind, i)
    L.params_destroy(P)


def check_sub_draws(L, kind, seed):
    q = common.pg(L).order
    P, po = common.make_params(L, seed, 8)
    d = synth.Drbg(seed, 'sub-draws-' + kind)
    vals, rs = sub_statement(L, kind, d)
    nd = 3 if kind == 'equality' else 7
    base = synth.random_tape(1, 32 * nd, seed=seed + 1)[0]
    cases = [(j, v) for j in range(nd) for v in (q, (1 << 256) - 1, 0, 1, q - 1)]
    if kind == 'mult' and getattr(L, 'group', 'tomEdwards256') == 'war256':
        # k_x = 0 makes A4_2 = Cy*k_x the identity, which war256 encodes in 1 byte (weier.ts:244-247) and a proof slot
        # cannot hold
        cases.remove((0, 0))
    tape = np.repeat(base[None, :], len(cases), axis=0)
    for i, (j, v) in enumerate(cases):
        tape[i, 32 * j:32 * j + 32] = np.frombuffer(i32(v), np.uint8)
    row = b''.join(i32(v) for v in vals + rs)
    com, proofs, st = L.prove_sub_batch(kind, P, arr([row] * len(cases)), tape)
    for i, (j, v) in enumerate(cases):
        if v >= q:
            assert st[i] == TAPE_RANGE and not proofs[i].any() and not com[i].any(), (kind, j, hex(v))
        else:
            want = sub_oracle(L, po, kind, vals, rs, tape[i])
            assert st[i] == 0 and proofs[i].tobytes() == want[0] and com[i].tobytes() == want[1], (kind, j, hex(v))
    L.params_destroy(P)


@pytest.mark.parametrize('kind', ['equality', 'mult'])
def test_sub_statement_scalars_host(hostsim, kind):
    check_sub_statement_scalars(hostsim, kind, seed=301)


@pytest.mark.parametrize('kind', ['equality', 'mult'])
def test_sub_statement_scalars_host_war256(hostsim_war, kind):
    check_sub_statement_scalars(hostsim_war, kind, seed=302)


@pytest.mark.parametrize('kind', ['equality', 'mult'])
def test_sub_draws_host(hostsim, kind):
    check_sub_draws(hostsim, kind, seed=303)


@pytest.mark.parametrize('kind', ['equality', 'mult'])
def test_sub_draws_host_war256(hostsim_war, kind):
    check_sub_draws(hostsim_war, kind, seed=304)


# ------------------------------------------------------------------------------ P-256 decoding
def enc(tag, x, y):
    return bytes([tag]) + i32(x) + i32(y)


def small_point():
    x, y = common.small_x_point(p256)
    return p256.deserialize_point(enc(4, x, y))


def encoding(label, pt):
    """label -> the 65-byte encoding; 'x+p' encodes small_point() (the only points whose x + p fits 32 bytes), every
    other label is built from pt"""
    if label == 'x+p':
        return common.noncanonical_enc(p256, *small_point().to_affine())
    x, y = pt.to_affine()
    return {'canonical': enc(4, x, y), 'zeros': bytes(65), 'tag00': enc(0, x, y), 'tag02': enc(2, x, y),
            'y+1': enc(4, x, y + 1)}[label]


def point_of(label, pt):
    return small_point() if label == 'x+p' else pt


def check_prove_pk(L, seed, sec=8):
    P, po = common.make_params(L, seed, sec)
    wl = synth.Workload(B=len(LABELS), N=4, seed=seed)
    for b, label in enumerate(LABELS):
        wl.pk[b] = np.frombuffer(encoding(label, p256.deserialize_point(wl.pk[b].tobytes())), np.uint8)
    tape = synth.random_tape(wl.B, L.prove_tape_len(wl.N, sec), seed=seed + 1)
    proofs, plen, st = common.run_prove(L, P, wl, tape, sec)
    for b, label in enumerate(LABELS):
        if label in BAD:
            assert st[b] == INVALID_PK and plen[b] == 0 and not proofs[b].any(), (label, st[b])
        else:
            pr, _ = common.oracle_proof(po, wl, tape, b)
            assert st[b] == 0 and proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), label
    L.params_destroy(P)


def check_prove_exp_points(L, seed, sec=6):
    """the base and Q of proveExp alone; the other point of each row is canonical"""
    P, po = common.make_params(L, seed, sec)
    d = synth.Drbg(seed, 'exp-points')
    G = p256.generator()
    rnd_pt = lambda: G.mul(p256.new_scalar(d.below(p256.order)))   # noqa: E731
    rows = []   # (site, label, base point, base bytes, Q point or None, Q bytes, s)
    for site in ('base', 'Q'):
        for label in LABELS:
            s, base, Q = d.below(p256.order), rnd_pt(), rnd_pt()
            bb, qb = flat._pt(base, 65), flat._pt(Q, 65)
            if site == 'base':
                bb, base = encoding(label, base), point_of(label, base)
            else:
                qb, Q = encoding(label, Q), (None if label == 'zeros' else point_of(label, Q))
            rows.append((site, label, base, bb, Q, qb, s))
    B = len(rows)
    tape = synth.random_tape(B, 32 * (3 + 4 * sec + 40 * sec), seed=seed + 1)
    pks = []
    for _, _, base, _, Q, _, s in rows:
        pk = base.mul(p256.new_scalar(s))
        pks.append(flat._pt(pk.sub(Q) if Q is not None else pk, 65))
    proofs, plen, st = L.prove_exp_batch(P, arr([r[3] for r in rows]), arr([i32(r[6]) for r in rows]), arr(pks),
                                         arr([r[5] for r in rows]), tape, sec)
    for b, (site, label, base, _, Q, _, s) in enumerate(rows):
        if label in BAD and not (site == 'Q' and label == 'zeros'):   # 65 zero bytes as Q: no Q
            assert st[b] == INVALID_PK and plen[b] == 0, (site, label, st[b])
            continue
        tp = Tape(tape[b].tobytes())
        x, y = p256.deserialize_point(pks[b]).to_affine()
        nist = OC.PedersenParams(p256, base, po.NistGroup.h)
        Cs = nist.commit(s, tp)
        Cx, Cy = po.ProofGroup.commit(x, tp), po.ProofGroup.commit(y, tp)
        pi = OE.prove_exp(nist, po.ProofGroup, s, Cs, p256.deserialize_point(pks[b]), Cx, Cy, sec, tp, Q)
        assert st[b] == 0 and proofs[b, :plen[b]].tobytes() == b''.join(flat.ser_exp(e) for e in pi), (site, label)
    L.params_destroy(P)


def check_prove_pointadd_points(L, seed):
    """P, Q and R of provePointAdd alone, each in turn given with every label (R = P + Q throughout)"""
    g = common.pg(L)
    P_, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    d = synth.Drbg(seed, 'padd-points')
    G = p256.generator()
    rnd_pt = lambda: G.mul(p256.new_scalar(d.below(p256.order)))   # noqa: E731
    rows = [('-', 'canonical')] + [(pos, label) for pos in range(3) for label in LABELS[1:]]
    B = len(rows)
    tape = synth.random_tape(B, 32 * 38, seed=seed + 1)
    bl = synth.random_tape(B, 32 * 6, seed=seed + 2)
    pts, want = [], []
    for b, (pos, label) in enumerate(rows):
        Pp, Qp = rnd_pt(), rnd_pt()
        if pos == 0:
            Pp = point_of(label, Pp)
        elif pos == 1:
            Qp = point_of(label, Qp)
        Rp = Pp.add(Qp)
        if pos == 2 and label == 'x+p':   # R is the small point: P = R - Q
            Rp = small_point()
            Pp = Rp.sub(Qp)
        three = [Pp, Qp, Rp]
        encs = [flat._pt(p, 65) for p in three]
        if pos != '-':
            encs[pos] = encoding(label, three[pos])
        pts.append(b''.join(encs))
        if label in BAD:
            want.append(None)
            continue
        r = [int.from_bytes(bl[b, 32 * i:32 * i + 32].tobytes(), 'big') for i in range(6)]
        coords = [c for p in three for c in p.to_affine()]
        cs = [OC.Commitment(params.h.dblmul(g.new_scalar(rr), params.g, g.new_scalar(v)), g.new_scalar(rr))
              for v, rr in zip(coords, r)]
        pi = OE.prove_point_add(params, Pp, Qp, Rp, *cs, Tape(tape[b].tobytes()))
        want.append((flat.ser_point_add(pi), b''.join(c.p.to_bytes() for c in cs)))
    com, proofs, st = L.prove_sub_batch('pointadd', P_, arr(pts), tape, bl)
    for b, (pos, label) in enumerate(rows):
        if want[b] is None:
            assert st[b] == INVALID_PK and not proofs[b].any() and not com[b].any(), (pos, label, st[b])
        else:
            assert st[b] == 0 and proofs[b].tobytes() == want[b][0] and com[b].tobytes() == want[b][1], (pos, label)
    L.params_destroy(P_)


def check_parse_points_ops(L, seed):
    """keyToInt (status per row) and the base of p256_mul_batch (no status: an invalid base stands for G, the identity
    base gives the identity)"""
    d = synth.Drbg(seed, 'parse-points')
    G = p256.generator()
    pts = [G.mul(p256.new_scalar(d.below(p256.order))) for _ in LABELS]
    encs = arr([encoding(label, pt) for label, pt in zip(LABELS, pts)])
    xs, st = L.key_to_int(encs)
    for i, label in enumerate(LABELS):
        if label in BAD:
            assert st[i] == INVALID_PK, (label, st[i])
        else:
            assert st[i] == 0 and int.from_bytes(xs[i].tobytes(), 'big') == point_of(label, pts[i]).to_affine()[0], label
    ks = [d.below(p256.order) for _ in LABELS]
    out = L.p256_mul_batch(encs, common.be(ks, 32))
    for i, label in enumerate(LABELS):
        if label == 'zeros':
            want = bytes(65)
        else:
            want = (G if label in BAD else point_of(label, pts[i])).mul(p256.new_scalar(ks[i])).to_bytes()
        assert out[i].tobytes() == want, label


def test_prove_pk_host(hostsim):
    check_prove_pk(hostsim, seed=311)


def test_prove_pk_host_war256(hostsim_war):
    check_prove_pk(hostsim_war, seed=312)


def test_prove_exp_points_host(hostsim):
    check_prove_exp_points(hostsim, seed=313)


def test_prove_exp_points_host_war256(hostsim_war):
    check_prove_exp_points(hostsim_war, seed=314)


def test_prove_pointadd_points_host(hostsim):
    check_prove_pointadd_points(hostsim, seed=315)


def test_prove_pointadd_points_host_war256(hostsim_war):
    check_prove_pointadd_points(hostsim_war, seed=316)


def test_parse_points_ops_host(hostsim):
    check_parse_points_ops(hostsim, seed=317)


def test_parse_points_ops_host_war256(hostsim_war):
    check_parse_points_ops(hostsim_war, seed=318)


@pytest.mark.gpu
@pytest.mark.parametrize('group', ['tomEdwards256', 'war256'])
def test_prove_sigma_edges_device(gpu_engine, gpu_engine_war, group):
    L = (gpu_engine if group == 'tomEdwards256' else gpu_engine_war).lib
    s = 320 if group == 'tomEdwards256' else 340
    for kind in ('equality', 'mult'):
        check_sub_statement_scalars(L, kind, seed=s + 1)
        check_sub_draws(L, kind, seed=s + 2)
    check_prove_pk(L, seed=s + 3)
    check_prove_exp_points(L, seed=s + 4)
    check_prove_pointadd_points(L, seed=s + 5)
    check_parse_points_ops(L, seed=s + 6)
