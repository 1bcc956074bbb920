"""Exact status codes of rows with one or several defects, against the reference's first throw.

`status[i]` mirrors the reference's throw sites (include/zkattest.h), and the host shims turn each code back into the
reference's error message, so a row with several defects must report the defect the reference meets FIRST:
  verifySignatureList (zkpAttestList.ts:147-184):  the whole proof parses (9), then R at infinity (8), then
  verifyMembership (a GK draw out of range: 5; false: ok = 0 and no code at all), then verifyExp: the index draws (5),
  then the sampled repetitions in sample order, each one 'params not found' (10), its first draw (5), T / T1 at
  infinity (2 / 3), its other draws (5).
The catalogue below builds each defect so that it hits a chosen sampled repetition (the sample order is
generateIndices on the verifier tape, exp.ts:95-109), and every row — each defect alone, ordered pairs in both sample
orders, some triples — is compared, exactly, with oracle/cpu (which throws in the reference's order) and with the
Python oracle wherever it applies (it redraws where the library reports ZKA_ERR_TAPE_RANGE, so rows with tape defects
are checked against oracle/cpu only).
"""
import itertools

import numpy as np
import pytest

import common
from oracle import exp as OE
from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from oracle.curves import p256
from zkp_ecdsa_b200 import synth, verify_tape as VT

S, N = 20, 5                      # SecLevel, ring size (depth 3)
NP = 65
PY_CODES = {'R is at infinity': 8, 'params not found': 10, 'T is at infinity': 2, 'T[i] is at infinity': 2,
            'T1 is at infinity': 3, "Points don't add up!": 4, 'invalid public key': 1}
T1_BASE = 7                       # a T1 defect replaces R by 7 G, so that the z making T1 the identity is known


@pytest.fixture(scope='module')
def cpu_port():
    import __graft_entry__ as g
    g.build_oracle_cpu()
    from zkp_ecdsa_b200.capi import ZkaLib
    return ZkaLib(g.ORACLE_CPU)


# ------------------------------------------------------------------------------------------------ the valid proof
class Base:
    """One valid proof of SecLevel S over a ring of N and a verifier tape for K samples; its repetitions, their
    challenge bits and the sample order of the tape."""

    def __init__(self, L, seed, K=S, sec=S, vt=None):
        self.L, self.K, self.S = L, K, sec
        self.P, self.po = common.make_params(L, seed, sec)
        self.wl = synth.Workload(B=1, N=N, seed=seed)
        tape = synth.random_tape(1, L.prove_tape_len(N, sec), seed=seed + 100)
        proofs, plen, st = common.run_prove(L, self.P, self.wl, tape, sec)
        assert st[0] == 0
        self.good = proofs[0, :plen[0]].tobytes()
        self.n = VT.ceil_log2(N)
        self.g = 32 * (2 * self.n + 1)
        self.vts = L.verify_tape_len_ex(N, sec, K)
        self.vt = vt if vt is not None else VT.random_verify_tape(1, self.vts, N, sec, seed=seed + 7)[0].tobytes()
        self.head = self.good[:flat.HEAD_LEN]
        self.reps, off = [], flat.HEAD_LEN
        for _ in range(sec):
            ln = flat.REP1_LEN if self.good[off] else flat.REP0_LEN
            self.reps.append(self.good[off:off + ln])
            off += ln
        self.gk = self.good[off:]
        self.bits = [r[0] for r in self.reps]        # the tag of a valid repetition is its challenge bit
        self.order = OE.generate_indices(K, sec, Tape(self.vt[self.g:self.g + sec - 2]))[:K]
        self.draw0, d = [], 0                        # first exp draw of each sample, 32-byte units
        for i in self.order:
            self.draw0.append(d)
            d += 3 if self.bits[i] else 25
        self.msg = self.wl.msg_hash[0].tobytes()
        self.ring_ints = self.wl.ring_ints()

    def close(self):
        self.L.params_destroy(self.P)     # its fixed-base tables are large: one set at a time on the device

    def samples_with(self, bit=None):
        return [j for j, i in enumerate(self.order) if bit is None or self.bits[i] == bit]


# ------------------------------------------------------------------------------------------------ the catalogue
# kind -> (code the defect gives alone, needs a sampled repetition with this challenge bit (None: any), python oracle
# applies).  Sample-targeted kinds take the sample position j; the others ignore it.
KINDS = {
    'r_inf': (8, None, True),         # R = the P-256 identity (65 zero bytes)
    'hdr_pt': (9, None, True),        # keyXcom off the curve
    'rep_pt': (9, None, True),        # Ty of a repetition off the curve
    'rep_sc': (9, None, True),        # alpha / z of a repetition >= p256.n
    'bad_tag': (9, None, True),       # a repetition tag of 2
    'gk_pt': (9, None, True),         # GK cl[0] off the curve
    'gk_sc': (9, None, True),         # GK zd >= the proof group's order
    'trunc': (9, None, True),         # last byte missing
    'trail': (9, None, True),         # one byte too many
    'gk_false': (0, None, True),      # zd + 1: verifyMembership returns false
    'gk_tape': (5, None, False),      # the first GK draw out of range
    'idx_tape': (5, None, False),     # the first generateIndices byte out of range
    'T': (2, 1, True),                # alpha = 0 in a bit-1 repetition: T is at infinity
    'T1': (3, 0, True),               # R = 7 G and z = -z1 / 7 in a bit-0 repetition: T1 is at infinity
    'tag': (10, None, True),          # the repetition re-serialised in the other tag's form: params not found
    'draw': (5, None, False),         # the sample's first exp draw (relA) out of range
}
SAMPLED = ('T', 'T1', 'tag', 'draw')
CONFLICTS = ({'r_inf', 'T1'}, {'trunc', 'trail'})


def build_row(base, defects):
    """(proof bytes, verifier tape row, python oracle applies) of the valid proof with `defects` [(kind, j)]."""
    head = bytearray(base.head)
    reps = [bytearray(r) for r in base.reps]
    gk = bytearray(base.gk)
    tape = bytearray(base.vt)
    ws, wp = flat.WS, flat.WP
    body = 1 + NP + 2 * wp                              # offset of the first body scalar (alpha / z)
    one = next(r for r in base.reps if r[0] == 1)
    zero = next(r for r in base.reps if r[0] == 0)
    trunc = trail = False
    py = True
    for kind, j in defects:
        i = base.order[j] if j is not None else 0
        py = py and KINDS[kind][2]
        if kind == 'r_inf':
            head[:NP] = bytes(NP)
        elif kind == 'hdr_pt':
            head[2 * NP + wp - 1] ^= 1
        elif kind == 'rep_pt':
            reps[i][1 + NP + 2 * wp - 1] ^= 1
        elif kind == 'rep_sc':
            reps[i][body:body + 32] = b'\xff' * 32
        elif kind == 'bad_tag':
            reps[i][0] = 2
        elif kind == 'gk_pt':
            gk[1 + wp - 1] ^= 1
        elif kind == 'gk_sc':
            gk[-ws:] = b'\xff' * ws
        elif kind == 'gk_false':
            gk[-1] ^= 1
        elif kind == 'trunc':
            trunc = True
        elif kind == 'trail':
            trail = True
        elif kind == 'gk_tape':
            tape[:32] = b'\xff' * 32
        elif kind == 'idx_tape':
            tape[base.g] = 0xff
        elif kind == 'draw':
            o = base.g + VT.IDX_PAD + 32 * base.draw0[j]
            tape[o:o + 32] = b'\xff' * 32
        elif kind == 'T':
            assert base.bits[i] == 1
            reps[i][body:body + 32] = bytes(32)
        elif kind == 'T1':
            assert base.bits[i] == 0
            n = p256.order
            R = p256.generator().mul(p256.new_scalar(T1_BASE))
            head[:NP] = R.to_bytes()
            z = OZ.truncate_to_n(int.from_bytes(base.msg, 'big'), n)
            z1 = pow(R.to_affine()[0] % n, -1, n) * z % n
            reps[i][body:body + 32] = (-z1 * pow(T1_BASE, -1, n) % n).to_bytes(32, 'big')
        elif kind == 'tag':
            other = zero if reps[i][0] else one      # the other tag with a body that parses
            reps[i] = bytearray(bytes([other[0]]) + bytes(reps[i][:body])[1:] + other[body:])
        else:
            raise AssertionError(kind)
    p = bytes(head) + b''.join(bytes(r) for r in reps) + bytes(gk)
    if trunc:
        p = p[:-1]
    if trail:
        p = p + b'\x00'
    return p, bytes(tape), py


def catalogue(base, triples=True):
    """[(label, defects)]: every kind alone (sampled kinds at two positions), every pair of kinds with the sampled
    ones in both sample orders, and a few triples."""
    def first(kind, after=-1, before=None):
        bit = KINDS[kind][1]
        for j in base.samples_with(bit):
            if j > after and (before is None or j < before):
                return j
        return None

    rows = []
    for kind in KINDS:
        if kind in SAMPLED:
            js = base.samples_with(KINDS[kind][1])
            for j in (js[0], js[len(js) // 2]):
                rows.append(((kind, j),))
        else:
            rows.append(((kind, None),))
    for a, b in itertools.combinations(KINDS, 2):
        if {a, b} in CONFLICTS:
            continue
        if a in SAMPLED and b in SAMPLED:
            ja = first(a)
            jb = first(b, after=ja)                      # a sampled before b
            if jb is not None:
                rows.append(((a, ja), (b, jb)))
            jb = first(b)
            ja = first(a, after=jb)                      # b sampled before a
            if ja is not None:
                rows.append(((a, ja), (b, jb)))
        else:
            rows.append(tuple((k, first(k) if k in SAMPLED else None) for k in (a, b)))
    for kind in ('T', 'T1', 'tag'):                      # the same defect at two samples
        js = base.samples_with(KINDS[kind][1])
        if len(js) > 1:
            rows.append(((kind, js[1]), (kind, js[0])))
    if triples:
        jt, jt1, jg = first('T'), first('T1'), first('tag')
        for trip in (
                (('T', jt), ('T1', jt1), ('tag', jg)),
                (('r_inf', None), ('hdr_pt', None), ('T', jt)),
                (('r_inf', None), ('gk_false', None), ('tag', jg)),
                (('gk_false', None), ('T', jt), ('tag', jg)),
                (('idx_tape', None), ('gk_false', None), ('T1', jt1)),
                (('gk_tape', None), ('T', jt), ('r_inf', None)),
                (('draw', first('draw', after=max(jt, jg))), ('T', jt), ('tag', jg)),
                (('gk_tape', None), ('idx_tape', None), ('draw', 0))):
            rows.append(trip)
    return [(' + '.join(f'{k}@{j}' if j is not None else k for k, j in r), r) for r in rows]


# ------------------------------------------------------------------------------------------------ expected codes
def python_expect(base, proof, tape):
    """(ok, code) of the Python oracle: a throw of flat.de_proof is a deserialisation error (9), the others map
    through their messages."""
    try:
        prf = flat.de_proof(proof, base.S)
    except ValueError:
        return 0, 9
    try:
        ok = OZ.verify_signature_list(base.po, base.msg, base.ring_ints, prf,
                                      Tape(VT.oracle_stream(tape, N, base.S)), base.K)
    except ValueError as e:
        return 0, PY_CODES[str(e)]
    return int(ok), 0


def pack(base, rows, ps=None):
    """rows [(proof, tape)] -> proofs, lens, tapes, msgs arrays of one batch"""
    ps = ps or base.L.proof_max_len(N, base.S) + 1
    B = len(rows)
    proofs = np.zeros((B, ps), np.uint8)
    lens = np.zeros(B, np.uint32)
    tapes = np.zeros((B, base.vts), np.uint8)
    for k, (p, t) in enumerate(rows):
        proofs[k, :len(p)] = np.frombuffer(p, np.uint8)
        lens[k] = len(p)
        tapes[k] = np.frombuffer(t, np.uint8)
    msgs = np.repeat(base.wl.msg_hash[:1], B, axis=0)
    return proofs, lens, tapes, msgs


def verify_rows(L, P, base, rows):
    proofs, lens, tapes, msgs = pack(base, rows)
    B = len(rows)
    ok = np.zeros(B, np.uint8)
    st = np.zeros(B, np.int32)
    L.verify_batch_ex(P, B, msgs, base.wl.ring, N, proofs, proofs.shape[1], lens, tapes, base.vts, ok, st, base.K)
    return [(int(a), int(b)) for a, b in zip(ok, st)]


def cpu_params(cpu, base, seed):
    hn, hp = cpu.params_generate(synth.params_rnd(seed))
    return cpu.params_create(hn, hp, base.S)


def expected(base, cat, cpu=None, cpu_P=None):
    """[(ok, code)] of every catalogue row: oracle/cpu and the Python oracle agree with each other where both apply."""
    built = [build_row(base, d) for _, d in cat]
    want = verify_rows(cpu, cpu_P, base, [(p, t) for p, t, _ in built]) if cpu is not None else [None] * len(cat)
    out = []
    for (label, defects), (p, t, py), w in zip(cat, built, want):
        if py:
            e = python_expect(base, p, t)
            assert w is None or w == e, (label, 'oracle/cpu', w, 'python', e)
            w = e
        assert w is not None, label
        if len(defects) == 1:                           # the catalogue builds what it says
            assert w[1] == KINDS[defects[0][0]][0] and (w[0] == 0), (label, w)
        out.append(w)
    return built, out


# ------------------------------------------------------------------------------------------------ tests
_cache = {}   # the catalogue and its expected codes, per proof group and setting (the oracles are slow)


def _setup(L, cpu, seed, K=S, sec=S, triples=True):
    """(base, catalogue, rows, expected codes) on library L; the caller closes base"""
    base = Base(L, seed, K=K, sec=sec)
    key = (getattr(L, 'group', 'tomEdwards256'), cpu is None, seed, K, sec, triples)
    if key not in _cache:
        cat = catalogue(base, triples)
        if cpu is None:
            cat = [(label, d) for label, d in cat if all(KINDS[k][2] for k, _ in d)]
        cP = cpu_params(cpu, base, seed) if cpu is not None else None
        built, want = expected(base, cat, cpu, cP)
        if cP is not None:
            cpu.params_destroy(cP)
        _cache[key] = (base.good, cat, built, want)
    good, cat, built, want = _cache[key]
    assert base.good == good
    return base, cat, built, want


def check_catalogue(L, cpu, seed, K=S, sec=S, triples=True, one_by_one=True, mixed_runs=1):
    """the rows one at a time, in one batch, and in one batch mixed with valid rows (`mixed_runs` times)"""
    base, cat, built, want = _setup(L, cpu, seed, K, sec, triples)
    try:
        rows = [(p, t) for p, t, _ in built]
        bad = []
        if one_by_one:
            for (label, _), r, w in zip(cat, rows, want):
                g = verify_rows(L, base.P, base, [r])[0]
                if g != w:
                    bad.append(('alone', label, g, w))
        got = verify_rows(L, base.P, base, rows)
        bad += [('batch', label, g, w) for (label, _), g, w in zip(cat, got, want) if g != w]
        assert not bad, '\n'.join(map(str, bad))
        if mixed_runs:
            check_mixed(L, base, cat, rows, want, runs=mixed_runs)
    finally:
        base.close()


def test_confirmed_cases(hostsim, cpu_port):
    """The two precedence bugs: a parse error behind R at infinity, and exp-side codes out of sample order."""
    base = Base(hostsim, 301)
    cP = cpu_params(cpu_port, base, 301)
    ones = [(('T', j),) for j in base.samples_with(1)]
    zeros = [(('tag', j),) for j in base.samples_with(0)]
    assert base.bits[base.order[0]] == 1              # the first sample is a bit-1 repetition: T is met first
    cases = {
        'R at infinity + off-curve keyXcom': ((('r_inf', None), ('hdr_pt', None)), (0, 9)),
        'alpha = 0 in every bit-1 repetition + every bit-0 repetition in tag-1 form':
            (sum(ones, ()) + sum(zeros, ()), (0, 2)),
    }
    for label, (defects, want) in cases.items():
        p, t, _ = build_row(base, defects)
        assert python_expect(base, p, t) == want, label
        assert verify_rows(cpu_port, cP, base, [(p, t)]) == [want], label
        assert verify_rows(hostsim, base.P, base, [(p, t)]) == [want], label
    cpu_port.params_destroy(cP)
    base.close()


def test_catalogue_hostsim(hostsim, cpu_port):
    check_catalogue(hostsim, cpu_port, 301)


def test_catalogue_hostsim_war256(hostsim_war):
    """war256 has no oracle/cpu build: the Python oracle rows only."""
    check_catalogue(hostsim_war, None, 311, triples=False, one_by_one=False)


# ------------------------------------------------------------------------------------------------ paths
def mixed_batch(L, base, rows, want, host_buffers=True):
    """The rows in one batch with valid rows at 0, 127, 128, the last row of the first chunk and the last row."""
    B = max(len(rows) + 5, 140)
    off = L.chunk_schedule(B, host_buffers)
    valid = {0, 127, 128, off[1] - 1, B - 1}
    vp, vt = base.good, base.vt
    out_rows, out_want, k = [], [], 0
    for b in range(B):
        if b in valid or k >= len(rows):
            out_rows.append((vp, vt))
            out_want.append((1, 0))
        else:
            out_rows.append(rows[k])
            out_want.append(want[k])
            k += 1
    assert k == len(rows)
    return out_rows, out_want


def check_mixed(L, base, cat, rows, want, runs=1):
    mrows, mwant = mixed_batch(L, base, rows, want)
    labels = {}
    it = iter(label for label, _ in cat)
    for b, w in enumerate(mwant):
        labels[b] = 'valid' if w == (1, 0) and mrows[b][0] == base.good and mrows[b][1] == base.vt else next(it, '?')
    outs = [verify_rows(L, base.P, base, mrows) for _ in range(runs)]
    bad = [(b, labels[b], g, w) for b, (g, w) in enumerate(zip(outs[0], mwant)) if g != w]
    assert not bad, '\n'.join(map(str, bad))
    for o in outs[1:]:
        assert o == outs[0]


@pytest.mark.parametrize('K', [5, 80])
def test_sample_counts(hostsim, cpu_port, K):
    """zka_verify_batch_ex with 5 and 80 samples (SecLevel 20 and 80)."""
    sec = S if K <= S else K
    keep = ('r_inf', 'hdr_pt', 'gk_false', 'idx_tape', 'gk_tape') + SAMPLED
    base = Base(hostsim, 321 + K, K=K, sec=sec)
    cat = [(label, d) for label, d in catalogue(base, triples=K < S) if all(k in keep for k, _ in d)]
    cP = cpu_params(cpu_port, base, 321 + K)
    built, want = expected(base, cat, cpu_port, cP)
    got = verify_rows(hostsim, base.P, base, [(p, t) for p, t, _ in built])
    cpu_port.params_destroy(cP)
    base.close()
    bad = [(label, g, w) for (label, _), g, w in zip(cat, got, want) if g != w]
    assert not bad, '\n'.join(map(str, bad))


def check_seeded(L, cpu, seed):
    """zka_verify_batch_seeded: the proof-side defects, every row with the same seed (so the same sample order)."""
    seeds = np.frombuffer(synth.Drbg(seed, 'status-seed').bytes(32), np.uint8).reshape(1, 32).copy()
    vt = L.seed_tape(1, seeds, N, S, S)[0].tobytes()
    base = Base(L, seed, vt=vt)
    cat = [(label, d) for label, d in catalogue(base) if all(KINDS[k][2] for k, _ in d)]
    cP = cpu_params(cpu, base, seed) if cpu is not None else None
    built, want = expected(base, cat, cpu, cP)
    if cP is not None:
        cpu.params_destroy(cP)
    proofs, lens, _, msgs = pack(base, [(p, t) for p, t, _ in built])
    B = len(cat)
    ok = np.zeros(B, np.uint8)
    st = np.zeros(B, np.int32)
    L.verify_batch_seeded(base.P, B, msgs, base.wl.ring, N, proofs, proofs.shape[1], lens, np.repeat(seeds, B, axis=0), S,
                          ok, st)
    base.close()
    bad = [(label, (int(a), int(b)), w) for (label, _), a, b, w in zip(cat, ok, st, want) if (int(a), int(b)) != w]
    assert not bad, '\n'.join(map(str, bad))


def test_seeded_hostsim(hostsim, cpu_port):
    check_seeded(hostsim, cpu_port, 331)


def check_rings(L, cpu, seed):
    """zka_verify_batch_rings over a ring set of depths 3 and 4: the catalogue against the proof's own ring (row
    layout of depth 3) interleaved with rows against the deeper ring, where verifyMembership returns false (GK length
    mismatch) before any draw, whatever else the row carries."""
    base, cat, built, want = _setup(L, cpu, seed)
    cP = cpu_params(cpu, base, seed) if cpu is not None else None
    other = synth.Workload(B=1, N=9, seed=seed + 1).ring
    sizes = np.array([N, 9], np.uint32)
    keys = np.concatenate([base.wl.ring, other]).copy()
    n2 = VT.ceil_log2(9)
    vts = L.verify_tape_len_ex(9, S, S)
    deep = [(('gk_false', None),), (('T', base.samples_with(1)[0]),), (('tag', 0),), (('gk_tape', None),),
            (('idx_tape', None), ('draw', 0)), ()]
    rows, ring_of, wants, labels = [], [], [], []
    for (label, _), (p, t, _), w in zip(cat, built, want):
        rows.append((p, t))
        ring_of.append(0)
        wants.append(w)
        labels.append(label)
    for d in deep:
        p, t, _ = build_row(base, d)
        t2 = bytes(32 * (2 * n2 + 1) - base.g) + t          # the deeper ring's GK drains in front of the same tail
        if d and d[0][0] == 'gk_tape':
            t2 = b'\xff' * 32 + t2[32:]
        w = verify_rows_ring(cpu, cP, base, [(p, t2)], other, 9, vts)[0] if cpu is not None else (0, 0)
        assert w == (0, 0), (d, w)
        rows.append((p, t2))
        ring_of.append(1)
        wants.append(w)
        labels.append('deeper ring: ' + ' + '.join(k for k, _ in d))
    order = np.random.default_rng(seed).permutation(len(rows))
    rows = [rows[k] for k in order]
    ring_of = np.array([ring_of[k] for k in order], np.uint32)
    wants = [wants[k] for k in order]
    labels = [labels[k] for k in order]
    B = len(rows)
    ps = L.proof_max_len(9, S) + 1
    proofs = np.zeros((B, ps), np.uint8)
    lens = np.zeros(B, np.uint32)
    tapes = np.zeros((B, vts), np.uint8)
    for k, (p, t) in enumerate(rows):
        proofs[k, :len(p)] = np.frombuffer(p, np.uint8)
        lens[k] = len(p)
        tapes[k, :len(t)] = np.frombuffer(t, np.uint8)
    msgs = np.repeat(base.wl.msg_hash[:1], B, axis=0)
    R = L.rings_create(sizes, keys)
    ok = np.zeros(B, np.uint8)
    st = np.zeros(B, np.int32)
    L.verify_batch_rings(base.P, R, ring_of, B, msgs, proofs, ps, lens, tapes, vts, S, ok, st)
    L.rings_destroy(R)
    base.close()
    if cP is not None:
        cpu.params_destroy(cP)
    bad = [(label, (int(a), int(b)), w) for label, a, b, w in zip(labels, ok, st, wants) if (int(a), int(b)) != w]
    assert not bad, '\n'.join(map(str, bad))


def verify_rows_ring(L, P, base, rows, ring, n_ring, vts):
    B = len(rows)
    ps = L.proof_max_len(n_ring, S) + 1
    proofs = np.zeros((B, ps), np.uint8)
    lens = np.zeros(B, np.uint32)
    tapes = np.zeros((B, vts), np.uint8)
    for k, (p, t) in enumerate(rows):
        proofs[k, :len(p)] = np.frombuffer(p, np.uint8)
        lens[k] = len(p)
        tapes[k, :len(t)] = np.frombuffer(t, np.uint8)
    ok = np.zeros(B, np.uint8)
    st = np.zeros(B, np.int32)
    L.verify_batch_ex(P, B, np.repeat(base.wl.msg_hash[:1], B, axis=0), ring, n_ring, proofs, ps, lens, tapes, vts, ok, st,
                      base.K)
    return [(int(a), int(b)) for a, b in zip(ok, st)]


def test_rings_hostsim(hostsim, cpu_port):
    check_rings(hostsim, cpu_port, 301)


EXP_KINDS = ('rep_pt', 'rep_sc', 'bad_tag', 'idx_tape') + SAMPLED
GK_KINDS = ('gk_pt', 'gk_sc', 'gk_false', 'gk_tape')


def check_standalone(L, cpu, seed):
    """verifyExp and verifyMembership alone (zka_verify_exp_batch, zka_verify_membership_batch): the rows whose
    defects are all on their side give the codes of the whole verifier."""
    base, cat, built, want = _setup(L, cpu, seed)
    g, hl = base.g, flat.HEAD_LEN
    ex = [(label, p, t, w) for (label, d), (p, t, _), w in zip(cat, built, want) if all(k in EXP_KINDS for k, _ in d)]
    n = p256.order
    B = len(ex)
    cols = {k: np.zeros((B, ln), np.uint8) for k, ln in (('base', 65), ('com', 65), ('px', flat.WP), ('py', flat.WP),
                                                           ('q', 65))}
    body = np.zeros((B, S * flat.REP0_LEN), np.uint8)
    blen = np.zeros(B, np.uint32)
    tapes = np.zeros((B, len(base.vt) - g), np.uint8)
    for k, (_, p, t, _) in enumerate(ex):
        cols['base'][k] = np.frombuffer(p[:65], np.uint8)
        cols['com'][k] = np.frombuffer(p[65:130], np.uint8)
        cols['px'][k] = np.frombuffer(p[130:130 + flat.WP], np.uint8)
        cols['py'][k] = np.frombuffer(p[130 + flat.WP:hl], np.uint8)
        R = p256.deserialize_point(p[:65])
        z = OZ.truncate_to_n(int.from_bytes(base.msg, 'big'), n)
        z1 = pow(R.to_affine()[0] % n, -1, n) * z % n
        cols['q'][k] = np.frombuffer(p256.generator().mul(p256.new_scalar(z1)).to_bytes(), np.uint8)
        r = p[hl:len(p) - len(base.gk)]
        body[k, :len(r)] = np.frombuffer(r, np.uint8)
        blen[k] = len(r)
        tapes[k] = np.frombuffer(t[g:], np.uint8)
    ok, st = L.verify_exp_batch(base.P, cols['base'], cols['com'], cols['px'], cols['py'], cols['q'], body, blen, tapes, S)
    bad = [(label, (int(a), int(b)), w) for (label, _, _, w), a, b in zip(ex, ok, st) if (int(a), int(b)) != w]
    assert not bad, '\n'.join(map(str, bad))
    gk = [(label, p, t, w) for (label, d), (p, t, _), w in zip(cat, built, want) if all(k in GK_KINDS for k, _ in d)]
    B = len(gk)
    com = np.repeat(np.frombuffer(base.head[130:130 + flat.WP], np.uint8)[None, :], B, axis=0)
    proofs = np.zeros((B, len(base.gk) + 1), np.uint8)
    lens = np.zeros(B, np.uint32)
    tapes = np.zeros((B, g), np.uint8)
    for k, (_, p, t, _) in enumerate(gk):
        r = p[len(p) - len(base.gk):]
        proofs[k, :len(r)] = np.frombuffer(r, np.uint8)
        lens[k] = len(r)
        tapes[k] = np.frombuffer(t[:g], np.uint8)
    ok, st = L.verify_membership_batch(base.P, com, base.wl.ring, proofs, lens, tapes)
    base.close()
    bad = [(label, (int(a), int(b)), w) for (label, _, _, w), a, b in zip(gk, ok, st) if (int(a), int(b)) != w]
    assert not bad, '\n'.join(map(str, bad))


def test_standalone_hostsim(hostsim, cpu_port):
    check_standalone(hostsim, cpu_port, 301)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(params=['gpu_engine', 'gpu_engine_war'])
def gpu_lib(request):
    return request.getfixturevalue(request.param).lib


@pytest.mark.gpu
@pytest.mark.parametrize('lanes', [1, 3])
def test_catalogue_gpu(gpu_lib, cpu_port, lanes):
    """The catalogue alone and mixed with valid rows, 128-row chunks, 1 and 3 lanes; the multi-defect batch twice with
    identical status arrays (exp-side codes of one proof come from concurrent threads)."""
    L = gpu_lib
    cpu = cpu_port if L.group == 'tomEdwards256' else None
    old = L.config()
    L.set_option('lanes', lanes)
    L.set_option('chunk', 128)
    L.set_option('host_chunk', 128)
    try:
        check_catalogue(L, cpu, 301 if cpu is not None else 311, triples=cpu is not None, mixed_runs=2)
        if cpu is not None:
            check_seeded(L, cpu, 331)
            check_rings(L, cpu, 301)
            check_standalone(L, cpu, 301)
    finally:
        L.set_option('lanes', old['lanes'])
        L.set_option('chunk', old['chunk'])
        L.set_option('host_chunk', 2048)


# ------------------------------------------------------------------------------------------------ prover
PS = 16                           # prover SecLevel
DRAW_REP0 = 3                     # draws 3 + 4i .. 6 + 4i: alpha_i, r_i, Tx_i.r, Ty_i.r


def _nonce(wl, b=0):
    """the ECDSA nonce k of row b of a synth.Workload (replays its nonce stream)"""
    dn = synth.Drbg(wl.seed, 'nonces')
    r = int.from_bytes(wl.sig[b, :32].tobytes(), 'big')
    for _ in range(b + 1):
        k = dn.below(p256.order - 1) + 1
    assert p256.generator().mul(p256.new_scalar(k)).to_affine()[0] % p256.order == r
    return k


class ProveBase:
    def __init__(self, L, seed):
        self.L = L
        self.P, self.po = common.make_params(L, seed, PS)
        self.wl = synth.Workload(B=1, N=N, seed=seed)
        self.tl = L.prove_tape_len(N, PS)
        self.tape = synth.random_tape(1, self.tl, seed=seed + 100)[0].tobytes()
        n = p256.order
        r = int.from_bytes(self.wl.sig[0, :32].tobytes(), 'big')
        s = int.from_bytes(self.wl.sig[0, 32:].tobytes(), 'big')
        z = OZ.truncate_to_n(int.from_bytes(self.wl.msg_hash[0].tobytes(), 'big'), n)
        rinv = pow(r, -1, n)
        # alpha = s1 - z1 / k makes z = alpha - s1 = -z1 / k and T1 = z R + Q = -z1 G + z1 G the identity
        self.alpha_t1 = (rinv * s - rinv * z * pow(_nonce(self.wl), -1, n)) % n

    def row(self, defects):
        pk, which = self.wl.pk[0].copy(), int(self.wl.which[0])
        t = bytearray(self.tape)
        for kind, i in defects:
            if kind == 'pk':
                pk[40] ^= 1
            elif kind == 'which':
                which = N + 3
            elif kind == 'T':
                t[32 * (DRAW_REP0 + 4 * i):32 * (DRAW_REP0 + 4 * i + 1)] = bytes(32)
            elif kind == 'T1':
                t[32 * (DRAW_REP0 + 4 * i):32 * (DRAW_REP0 + 4 * i + 1)] = self.alpha_t1.to_bytes(32, 'big')
            elif kind == 'range':
                t[32 * i:32 * i + 32] = b'\xff' * 32
            else:
                raise AssertionError(kind)
        return pk, which, bytes(t)

    def python(self, defects):
        if any(k in ('which', 'range') for k, _ in defects):
            return None                     # the oracle redraws / has no ring-index check of its own
        pk, which, t = self.row(defects)
        try:
            p256.deserialize_point(pk.tobytes())
        except ValueError:
            return 1
        try:
            OZ.prove_signature_list(self.po, self.wl.msg_hash[0].tobytes(), self.wl.sig[0].tobytes(), pk.tobytes(), which,
                                    self.wl.ring_ints(), Tape(t))
        except ValueError as e:
            return PY_CODES[str(e)]
        return 0


def prove_rows(L, P, pb, rows):
    B = len(rows)
    wl = synth.Workload(B=1, N=N, seed=pb.wl.seed)
    msg = np.repeat(wl.msg_hash[:1], B, axis=0)
    sig = np.repeat(wl.sig[:1], B, axis=0)
    pk = np.zeros((B, 65), np.uint8)
    which = np.zeros(B, np.uint32)
    tape = np.zeros((B, pb.tl), np.uint8)
    for k, d in enumerate(rows):
        pk[k], which[k], t = pb.row(d)
        tape[k] = np.frombuffer(t, np.uint8)
    ps = L.proof_max_len(N, PS)
    proofs = np.zeros((B, ps), np.uint8)
    plen = np.zeros(B, np.uint32)
    st = np.zeros(B, np.int32)
    L.prove_batch(P, B, msg, sig, pk, which, wl.ring, N, tape, pb.tl, proofs, ps, plen, st)
    return [int(v) for v in st]


def test_prover_codes(hostsim, cpu_port):
    """T[i] at infinity (alpha_i = 0), T1 at infinity (alpha_i = s1 - z1 / k in a bit-0 repetition), an invalid pk, a
    ring index outside the ring and draws out of range, alone and combined."""
    pb = ProveBase(hostsim, 341)
    i1 = next(i for i in range(2, PS) if pb.python([('T1', i)]) == 3)      # a repetition whose bit stays 0
    rows = [(('pk', None),), (('which', None),), (('T', 5),), (('T1', i1),), (('range', 0),), (('range', DRAW_REP0 + 4 * 9),),
            (('pk', None), ('T', 5)), (('which', None), ('T', 5)), (('pk', None), ('which', None)),
            (('T', 2), ('T', 7)), (('T', 7), ('T1', i1)), (('T', PS - 1), ('T1', i1)), (('which', None), ('T1', i1)),
            (('pk', None), ('range', 1)), (('which', None), ('range', 1))]
    hn, hp = cpu_port.params_generate(synth.params_rnd(341))
    cP = cpu_port.params_create(hn, hp, PS)
    want = prove_rows(cpu_port, cP, pb, rows)
    for d, w in zip(rows, want):
        py = pb.python(list(d))
        assert py is None or py == w, (d, 'oracle/cpu', w, 'python', py)
    got = prove_rows(hostsim, pb.P, pb, rows)
    bad = [(d, g, w) for d, g, w in zip(rows, got, want) if g != w]
    assert not bad, '\n'.join(map(str, bad))
    for d, g in zip(rows, got):
        assert prove_rows(hostsim, pb.P, pb, [d]) == [g], d
    cpu_port.params_destroy(cP)
    hostsim.params_destroy(pb.P)
