"""Forged rows against the chunk-wide aggregate check of the verifier (zk_verify_agg.cuh).

The aggregate sums the linear combinations (GK, multiW, multiN) of every row of a chunk and accepts the whole chunk when
the sums are the identity.  The verify tape is an input: rows may share a tape row (or a seed), and a prover may know the
tape.  Two rejected rows whose residuals (the amount by which a combination misses the identity) cancel in the sum must
still be rejected, and so must one row whose GK residual cancels its multiW residual.  Each case compares every row's
verdict and status with the same call under the per-proof path (aggregate off) and with the oracle's verdict on the row's
own tape, and checks that no chunk holding a rejected row is counted as decided by the aggregate.

Families (d: a shift, X: a point, rho: the randomizer the reference draws for a relation):
  1. shared tape row, opposite response shifts (zd, za, zb of the GK proof; beta2 of a sampled repetition in multiW;
     beta1 / z2 in multiN): every response here enters its combination linearly, as (h, +-response) * rho;
  2. shared tape row, opposite points injected into a commitment before the Fiat-Shamir hash (cd[0] of the GK proof,
     A_1 of an equality proof inside a point-add proof in multiW, A of a repetition in multiN);
  3. distinct tape rows, a prover who knows them: residual X*rho_A in row A, -X*rho_A in row B via a relation of rho_B;
  4. one row whose GK residual is cancelled by a multiW residual scaled by the ratio of the two randomizers;
  5. the seeded and the ring-set entry points.
The weights that close them must be bound to the rows' inputs: a model of the derivation, shown exact against the
library, lets forgers who leave inputs out of it (the proof bytes, the GK block, the repetitions, the header, all but the
row index) build rows that cancel under their model, and the library must still reject them.
"""
import numpy as np
import pytest

import common
from oracle import flat
from oracle import multimult as OM
from oracle import zkattest as OZ
from oracle.big import Tape
from oracle.curves import p256
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT

SEC = 20          # sec_level = samples: every repetition is sampled exactly once (generate_indices is a permutation)
N = 5
D = 12345


# ------------------------------------------------------------------------------------------------ the oracle's relations
def relations(po, msg, ring_ints, proof_bytes, vt_row, ring_size=N, sec=SEC):
    """Every relation the reference drains for this row on this tape: [(group, rho, [(point, scalar int)])], in order."""
    rec = []
    orig = OM.Relation.drain

    def drain(self, m):    # multimult.ts:168-173, recording the randomizer
        rho = self.group.random_scalar(self.tape)
        rec.append((self.group, rho.k, [(pr.pt, pr.scalar.k) for pr in self.pairs]))
        for pr in self.pairs:
            m.insert(pr.pt, pr.scalar.mul(rho))
    OM.Relation.drain = drain
    try:
        prf = flat.de_proof(proof_bytes, sec)
        OZ.verify_signature_list(po, msg, ring_ints, prf, Tape(VT.oracle_stream(vt_row, ring_size, sec)))
    finally:
        OM.Relation.drain = orig
    return rec


def rho_of(rels, group, scalar):
    """The randomizer of the one relation of `group` that holds `scalar` (mod the group order) as a coefficient."""
    hits = [r for g, r, prs in rels if g is group and any(s == scalar % group.order for _, s in prs)]
    assert len(hits) == 1, len(hits)
    return hits[0]


# ------------------------------------------------------------------------------------------------ response shifts
# (field, group of the scalar, sign with which the response enters its relation's coefficient of h)
def _resp(prf, field):
    """(getter, setter, group, sign) of a response scalar of the proof."""
    gk = prf.membershipProof
    rep1 = next(e for e in prf.expProof if e.alpha is not None)
    rep0 = next(e for e in prf.expProof if e.alpha is None)
    tom = flat.PROOF_GROUP
    table = {
        'zd': (gk, 'zd', None, tom, -1),           # gk.ts: rel_final (g, -total) (h, -zd)
        'za': (gk, 'za', 0, tom, -1),              # rel0 of bit 0: (h, -za[0])
        'zb': (gk, 'zb', 0, tom, -1),              # rel1 of bit 0: (h, -zb[0])
        'beta2': (rep1, 'beta2', None, tom, 1),    # exp.ts relTx: (g, sx) (h, beta2) (-Tx, 1)      -> multiW
        'beta1': (rep1, 'beta1', None, p256, 1),   # relA: (T, 1) (h, beta1) (-A, 1)                -> multiN
        'z2': (rep0, 'z2', None, p256, 1),         # relA: (T1, 1) (Clambda, 1) (-A, 1) (h, z2)     -> multiN
    }
    obj, name, idx, grp, sign = table[field]

    def get():
        v = getattr(obj, name)
        return (v[idx] if idx is not None else v).k

    def put(k):
        s = grp.new_scalar(k % grp.order)
        if idx is None:
            setattr(obj, name, s)
        else:
            getattr(obj, name)[idx] = s
    return get, put, grp, sign


def shifted(row, field, d, sec=SEC):
    """The proof bytes `row` with the response `field` shifted by d (mod its group order)."""
    prf = flat.de_proof(bytes(row), sec)
    assert flat.ser_proof(prf) == bytes(row)
    get, put, _, _ = _resp(prf, field)
    put(get() + d)
    return flat.ser_proof(prf)


def response_info(row, field):
    prf = flat.de_proof(bytes(row), SEC)
    get, _, grp, sign = _resp(prf, field)
    return get(), grp, sign


# ------------------------------------------------------------------------------------------------ injected points
def prove_with_injection(po, wl, tape, b, where, X):
    """The oracle's proof of row b with X added to one commitment BEFORE the Fiat-Shamir hash that covers it, so every
    other part of the proof is consistent with the altered commitment:
      'gk'  cd[0] of the GK proof (rel_final holds it with coefficient -x^0 = -1),
      'eq'  A_1 of every equality proof (inside the point-add proofs of the 0-bit repetitions: multiW)."""
    from oracle import commit as OC
    from oracle import exp as OE
    from oracle import gk as OG
    from oracle.big import rnd
    from oracle.curves import hash_points
    saved = (OG.gk_commit, OE.prove_equality)
    try:
        if where == 'gk':
            calls = [0]
            n = max(1, (wl.N - 1).bit_length())

            def gk_commit(params, val, blinder):
                calls[0] += 1
                pt = saved[0](params, val, blinder)
                return pt.add(X) if calls[0] == 3 * n + 1 else pt       # cl, ca, cb of every bit, then cd[0]
            OG.gk_commit = gk_commit
        else:
            def prove_equality(params, x, C1, C2, tp):      # equality.ts:60-78 with A_1 + X
                k = rnd(params.c.order, tp)
                A1 = params.commit(k, tp)
                A2 = params.commit(k, tp)
                A1p = A1.p.add(X)
                c = hash_points([C1.p, C2.p, A1p, A2.p])
                cc, xx, kk = params.c.new_scalar(c), params.c.new_scalar(x), params.c.new_scalar(k)
                return OC.EqualityProof(A1p, A2.p, kk.sub(cc.mul(xx)), A1.r.sub(cc.mul(C1.r)), A2.r.sub(cc.mul(C2.r)))
            OE.prove_equality = prove_equality
        return flat.ser_proof(common.oracle_proof(po, wl, tape, b)[0])
    finally:
        OG.gk_commit, OE.prove_equality = saved


# ------------------------------------------------------------------------------------------------ batches and cases
class Batch:
    """B valid rows proved by the library, their messages and verify tapes; forged rows are built from row 0."""

    def __init__(self, L, B, seed, sec=SEC, ring_size=N, vtape=None):
        self.L, self.B, self.sec, self.N, self.seed = L, B, sec, ring_size, seed
        self.P, self.po = common.make_params(L, seed, sec)
        self.wl = synth.Workload(B=B, N=ring_size, seed=seed)
        self.ptape = synth.random_tape(B, L.prove_tape_len(ring_size, sec), seed=seed + 100)
        self.proofs, self.plen, status = common.run_prove(L, self.P, self.wl, self.ptape, sec)
        assert not status.any()
        self.vts = L.verify_tape_len(ring_size, sec)
        self.vt = vtape if vtape is not None else VT.random_verify_tape(B, self.vts, ring_size, sec, seed=seed + 7)
        self.ring_ints = self.wl.ring_ints()
        self.row0 = self.proofs[0, :self.plen[0]].tobytes()
        self._verdicts = {}

    def close(self):
        self.L.params_destroy(self.P)

    def oracle(self, proof, msg, vt_row):
        key = (proof, msg, vt_row)
        if key not in self._verdicts:
            self._verdicts[key] = common.oracle_verdict(self.po, msg, self.ring_ints, proof, vt_row, self.N, self.sec)
        return self._verdicts[key]

    def assemble(self, forged):
        """forged: {row: (proof bytes, verify tape row)}; every forged row carries row 0's message."""
        msgs, arr, lens, vt = self.wl.msg_hash.copy(), self.proofs.copy(), self.plen.copy(), self.vt.copy()
        for i, (p, t) in forged.items():
            assert len(p) <= arr.shape[1]
            arr[i] = 0
            arr[i, :len(p)] = np.frombuffer(p, np.uint8)
            lens[i] = len(p)
            msgs[i] = self.wl.msg_hash[0]
            vt[i] = np.frombuffer(t, np.uint8)
        return msgs, arr, lens, vt


def verify_both(L, call, B, chunk=None, lanes=None):
    """call(ok, status) with the aggregate on, then off: (ok, status, agg_pass added, agg_fail added, ok_off, status_off)."""
    cfg = L.config()
    if chunk:
        L.set_option('chunk', chunk)
        L.set_option('host_chunk', chunk)
    if lanes:
        L.set_option('lanes', lanes)
    try:
        ok, st = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        p0, f0 = L.stat('agg_pass'), L.stat('agg_fail')
        call(ok, st)
        dp, df = L.stat('agg_pass') - p0, L.stat('agg_fail') - f0
        sched = L.chunk_schedule(B, host_buffers=True)
        L.set_option('agg', 1)
        ok2, st2 = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        call(ok2, st2)
    finally:
        L.set_option('agg', 2)
        if chunk:
            L.set_option('chunk', cfg['chunk'])
            L.set_option('host_chunk', 2048)
        if lanes:
            L.set_option('lanes', cfg['lanes'])
    return ok, st, dp, df, ok2, st2, sched


def check_counters(ok, st, dp, df, sched):
    """Every chunk is counted once; a chunk holding a rejected row is never counted as decided by the aggregate, and a
    chunk of valid rows always is."""
    bad = [any(ok[a:b] == 0) for a, b in zip(sched, sched[1:])]
    assert (dp, df) == (bad.count(False), bad.count(True)), (dp, df, sched, list(ok))


def check_call(L, call, B, rejected, chunk=None, lanes=None):
    """call(ok, status) verifies B rows; `rejected` maps each forged row to the oracle's verdict on its own tape, which
    must be False.  The verdicts and statuses equal the per-proof path's, the forged rows are rejected, the others
    accepted, and the aggregate counters agree with the chunks."""
    ok, st, dp, df, ok2, st2, sched = verify_both(L, call, B, chunk, lanes)
    assert (ok == ok2).all() and (st == st2).all(), (list(ok), list(ok2), list(st), list(st2))
    for i, verdict in rejected.items():
        assert verdict is False, (i, verdict)
        assert ok[i] == 0 and st[i] == 0, (i, int(ok[i]), int(st[i]))
    assert all(ok[i] == 1 and st[i] == 0 for i in range(B) if i not in rejected), list(ok)
    check_counters(ok, st, dp, df, sched)
    return ok, st


def cpu_verdicts(bt, cpu, rows, msgs, arr, lens, vt):
    """oracle/cpu (the C++ restatement of the reference) on each of the given rows in a call of its own: (ok, status)."""
    hn, hp = cpu.params_generate(synth.params_rnd(bt.seed))
    Pc = cpu.params_create(hn, hp, bt.sec)
    ok, st = np.zeros(len(rows), np.uint8), np.zeros(len(rows), np.int32)
    for k, i in enumerate(rows):
        sub = [np.ascontiguousarray(a[i:i + 1]) for a in (msgs, arr, lens, vt)]
        cpu.verify_batch(Pc, 1, sub[0], bt.wl.ring, bt.N, sub[1], arr.shape[1], sub[2], sub[3], vt.shape[1], ok[k:k + 1], st[k:k + 1])
    cpu.params_destroy(Pc)
    return ok, st


def run_case(bt, forged, chunk=None, lanes=None, cpu=None, python=True):
    """Verify the batch with `forged` rows in it (check_call).  The forged rows' verdicts come from the Python oracle and,
    given `cpu`, from oracle/cpu too (which also sees one valid row)."""
    L = bt.L
    msgs, arr, lens, vt = bt.assemble(forged)

    def call(ok, st):
        L.verify_batch(bt.P, bt.B, msgs, bt.wl.ring, bt.N, arr, arr.shape[1], lens, vt, vt.shape[1], ok, st)
    rejected = {i: bt.oracle(p, msgs[i].tobytes(), t) if python else None for i, (p, t) in forged.items()}
    if cpu is not None:
        rows = sorted(forged) + [next(i for i in range(bt.B) if i not in forged)]
        okc, stc = cpu_verdicts(bt, cpu, rows, msgs, arr, lens, vt)
        assert list(okc) == [0] * len(forged) + [1] and not stc.any(), (list(okc), list(stc))
        for i in forged:
            rejected[i] = False if rejected[i] is None else rejected[i]
    return check_call(L, call, bt.B, rejected, chunk, lanes)


def pair(bt, pa, pb, ia, ib, ta=None, tb=None):
    """rows ia, ib get proofs pa, pb; both read the tape row ta (row 0's by default) unless tb is given."""
    ta = ta if ta is not None else bt.vt[0].tobytes()
    return {ia: (pa, ta), ib: (pb, tb if tb is not None else ta)}


def placements(B):
    return [(0, B - 1), (B // 2 - 1, B // 2), (B - 1, 1)]


def all_share_one_tape(bt, chunk=None, lanes=None):
    """Non-regression: valid rows that all read tape row 0 are still decided by the aggregate."""
    vt = np.repeat(bt.vt[:1], bt.B, axis=0)

    def call(ok, st):
        bt.L.verify_batch(bt.P, bt.B, bt.wl.msg_hash, bt.wl.ring, bt.N, bt.proofs, bt.proofs.shape[1], bt.plen, vt, vt.shape[1],
                          ok, st)
    check_call(bt.L, call, bt.B, {}, chunk, lanes)


def cancel_shift(bt, fa, da, ta, fb, tb, row_a=None, row_b=None):
    """The shift of response fb (read on tape row tb) whose residual cancels the residual of fa shifted by da (tape row ta):
    sign_a da rho_a + sign_b db rho_b = 0 (mod the order of their common group)."""
    row_a, row_b = row_a or bt.row0, row_b or bt.row0
    msg = bt.wl.msg_hash[0].tobytes()
    va, ga, sa = response_info(row_a, fa)
    vb, gb, sb = response_info(row_b, fb)
    assert ga.order == gb.order
    q = ga.order
    ra = rho_of(relations(bt.po, msg, bt.ring_ints, row_a, ta, bt.N, bt.sec), ga, sa * va)
    rb = rho_of(relations(bt.po, msg, bt.ring_ints, row_b, tb, bt.N, bt.sec), gb, sb * vb)
    return -sa * da * ra * pow(sb * rb, -1, q) % q


# ------------------------------------------------------------------------------------------------ the families
FIELDS = ('zd', 'za', 'zb', 'beta2', 'beta1', 'z2')


def check_family1(L, B=8, seed=61, cs=(0, 4, 9, 13, 16), fields=FIELDS):
    """Shared tape row, opposite response shifts: row A has response + d, row B response - d, both on tape row 0."""
    bt = Batch(L, B, seed)
    try:
        pa, pb = shifted(bt.row0, 'zd', D), shifted(bt.row0, 'zd', -D)
        for c in cs:                         # the default window first: a forced one stays set on the context
            if c:
                L.set_option('agg_c', c)
            run_case(bt, pair(bt, pa, pb, 0, B - 1))
        for ia, ib in placements(B):
            run_case(bt, pair(bt, pa, pb, ia, ib))
        # A and B in different chunks: rejected too, and the chunks without them still pass
        for ch in (B // 2, 2):
            run_case(bt, pair(bt, pa, pb, 0, B - 1), chunk=ch)
        for f in fields[1:]:
            run_case(bt, pair(bt, shifted(bt.row0, f, D), shifted(bt.row0, f, -D), 1, B - 2))
        all_share_one_tape(bt)
        all_share_one_tape(bt, chunk=B // 2)
    finally:
        bt.close()


def check_family2(L, B=6, seed=71):
    """Shared tape row, opposite prime-order points injected into commitments: cd[0] of the GK proof, A_1 of the equality
    proofs in multiW (both hashed after the injection), comS1 in multiN (held by every 0-bit relA; no hash covers it)."""
    bt = Batch(L, B, seed)
    try:
        grp = bt.po.ProofGroup
        Xt = grp.g.mul(grp.c.new_scalar(D))
        Xn = bt.po.NistGroup.g.mul(p256.new_scalar(D))

        def with_coms1(X):
            prf = flat.de_proof(bt.row0, SEC)
            prf.comS1 = prf.comS1.add(X)
            return flat.ser_proof(prf)
        cases = [(prove_with_injection(bt.po, bt.wl, bt.ptape, 0, where, Xt),
                  prove_with_injection(bt.po, bt.wl, bt.ptape, 0, where, Xt.neg())) for where in ('gk', 'eq')]
        cases.append((with_coms1(Xn), with_coms1(Xn.neg())))
        for pa, pb in cases:
            for ia, ib in ((0, B - 1), (2, 3)):
                run_case(bt, pair(bt, pa, pb, ia, ib))
    finally:
        bt.close()


def check_family3(L, B=6, seed=75):
    """Distinct tape rows and a prover who knows them: row A's residual is cancelled by row B's through another
    randomizer (same relation kind, another relation kind, and GK against multiW across the two rows)."""
    bt = Batch(L, B, seed)
    try:
        ta, tb = bt.vt[0].tobytes(), bt.vt[B - 1].tobytes()
        for fa, fb in (('zd', 'zd'), ('beta1', 'z2'), ('zd', 'beta2'), ('za', 'zb')):
            db = cancel_shift(bt, fa, D, ta, fb, tb)
            pa, pb = shifted(bt.row0, fa, D), shifted(bt.row0, fb, db)
            for ia, ib in ((0, B - 1), (2, 3)):
                run_case(bt, pair(bt, pa, pb, ia, ib, ta, tb))
    finally:
        bt.close()


def check_family4(L, B=6, seed=77):
    """One row whose GK residual (zd + d) is cancelled by its own multiW residual (beta2 of a 1-bit repetition), scaled by
    the ratio of the two randomizers read from the row's tape.  The reference rejects it at verifyMembership."""
    bt = Batch(L, B, seed)
    try:
        for i in (0, B // 2, B - 1):
            t = bt.vt[i].tobytes()
            d2 = cancel_shift(bt, 'zd', D, t, 'beta2', t)
            p = shifted(shifted(bt.row0, 'zd', D), 'beta2', d2)
            run_case(bt, {i: (p, t)})
    finally:
        bt.close()


def check_seeded(L, B=6, seed=79):
    """Family 1 through zka_verify_batch_seeded: two rows with equal seeds."""
    bt = Batch(L, B, seed)
    try:
        pa, pb = shifted(bt.row0, 'zd', D), shifted(bt.row0, 'zd', -D)
        seeds = np.frombuffer(synth.Drbg(seed, 'agg-forged-seeds').bytes(32 * B), np.uint8).reshape(B, 32).copy()
        for ia, ib in placements(B):
            sd = seeds.copy()
            sd[ib] = sd[ia]
            tape = L.seed_tape(1, sd, bt.N, SEC, SEC)
            msgs, arr, lens, _ = bt.assemble({ia: (pa, tape[ia].tobytes()), ib: (pb, tape[ib].tobytes())})

            def call(ok, st):
                L.verify_batch_seeded(bt.P, B, msgs, bt.wl.ring, bt.N, arr, arr.shape[1], lens, sd, SEC, ok, st)
            rejected = {i: bt.oracle(p, msgs[i].tobytes(), tape[i].tobytes()) for i, p in ((ia, pa), (ib, pb))}
            check_call(L, call, B, rejected)
    finally:
        bt.close()


def check_ring_sets(L, seeded, seed=83, S=SEC):
    """Family 1 through zka_verify_batch_rings / _rings_seeded: the pair on a ring of depth 3 (row 0's), valid rows on a
    ring of depth 4 in the same chunk."""
    import test_rings as TR
    sizes, ring_of = [5, 9], [0, 1, 1, 0, 1, 0, 1]
    B = len(ring_of)
    wl = synth.RingsWorkload(B, sizes, ring_of, seed)
    P, po = common.make_params(L, seed, S)
    rs = TR.Set(L, wl)
    try:
        tape = synth.random_tape(B, L.prove_tape_len(max(sizes), S), seed=seed + 100)
        proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
        assert not st.any()
        row0 = proofs[0, :plen[0]].tobytes()
        pa, pb = shifted(row0, 'zd', D), shifted(row0, 'zd', -D)
        ia, ib = 3, 5
        msgs, arr, lens = wl.msg_hash.copy(), proofs.copy(), plen.copy()
        for i, p in ((ia, pa), (ib, pb)):
            arr[i] = 0
            arr[i, :len(p)] = np.frombuffer(p, np.uint8)
            lens[i] = len(p)
            msgs[i] = wl.msg_hash[0]
        if seeded:
            seeds = TR._seeds(B, f'agg-forged-{seed}')
            seeds[ib] = seeds[ia]
            vt = TR.row_seed_tape(L, 1, seeds, sizes, ring_of, S, S)

            def call(ok, st):
                L.verify_batch_rings_seeded(P, rs.h, np.array(ring_of, np.uint32), B, msgs, arr, arr.shape[1], lens, seeds, S,
                                            ok, st)
        else:
            vt = TR.row_verify_tape(sizes, ring_of, S, S, seed)
            vt[ib] = vt[ia]

            def call(ok, st):
                L.verify_batch_rings(P, rs.h, np.array(ring_of, np.uint32), B, msgs, arr, arr.shape[1], lens, vt, vt.shape[1], S,
                                     ok, st)
        ring0 = wl.ring_ints(0)
        rejected = {i: common.oracle_verdict(po, msgs[i].tobytes(), ring0, p, vt[i].tobytes(), sizes[0], S)
                    for i, p in ((ia, pa), (ib, pb))}
        check_call(L, call, B, rejected)
    finally:
        rs.close()
        L.params_destroy(P)


# ------------------------------------------------------------------------------------------------ host simulators
@pytest.fixture(params=['tom', 'war'])
def sim(request):
    return request.getfixturevalue('hostsim' if request.param == 'tom' else 'hostsim_war')


def test_shared_tape_opposite_shifts_hostsim(sim):
    check_family1(sim)


def test_shared_tape_injected_points_hostsim(sim):
    check_family2(sim)


def test_distinct_tapes_tape_aware_prover_hostsim(sim):
    check_family3(sim)


def test_gk_residual_cancelled_by_multiw_hostsim(sim):
    check_family4(sim)


def test_equal_seeds_hostsim(sim):
    check_seeded(sim)


@pytest.mark.parametrize('seeded', [False, True])
def test_ring_sets_hostsim(sim, seeded):
    check_ring_sets(sim, seeded)


# ------------------------------------------------------------------------------------------------ GPU
def _cpu_port():
    import os
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    assert os.path.exists(g.ORACLE_CPU), 'oracle/_ref/libzkattest_cpu.so missing: run build()'
    return ZkaLib(g.ORACLE_CPU)


@pytest.fixture(params=['tom', 'war'])
def gpu(request):
    return request.getfixturevalue('gpu_engine' if request.param == 'tom' else 'gpu_engine_war').lib


@pytest.mark.gpu
def test_forged_families_on_gpu(gpu):
    check_family1(gpu, cs=(0, 9, 13, 16))
    check_family2(gpu)
    check_family3(gpu)
    check_family4(gpu)
    check_seeded(gpu)
    check_ring_sets(gpu, False)
    check_ring_sets(gpu, True)


def check_lanes(L, cpu, lanes, B=300, seed=87):
    """128-row chunks on 1 or 3 lanes: the pair at the first and last row of a chunk, in the middle of one, and in two
    chunks; the oracle/cpu verdicts too."""
    bt = Batch(L, B, seed)
    try:
        pa, pb = shifted(bt.row0, 'zd', D), shifted(bt.row0, 'zd', -D)
        for ia, ib in ((0, 127), (60, 61), (0, B - 1)):
            run_case(bt, pair(bt, pa, pb, ia, ib), chunk=128, lanes=lanes, cpu=cpu)
        qa, qb = shifted(bt.row0, 'beta1', D), shifted(bt.row0, 'beta1', -D)
        run_case(bt, pair(bt, qa, qb, 200, 255), chunk=128, lanes=lanes, cpu=cpu)
        all_share_one_tape(bt, chunk=128, lanes=lanes)
    finally:
        bt.close()


@pytest.mark.gpu
@pytest.mark.parametrize('lanes', [1, 3])
def test_lanes_and_chunks_on_gpu(gpu, lanes):
    check_lanes(gpu, _cpu_port() if gpu.group == 'tomEdwards256' else None, lanes)   # oracle/cpu: tomEdwards256 only


@pytest.mark.gpu
@pytest.mark.parametrize('war', [False, True])
def test_full_chunk_on_gpu(war):
    """One chunk of 4096 rows over a ring of 256 at sec_level 80, on a fresh context (no window forced by an earlier test)
    so that the aggregate's cost model picks its own; the pair (zd + d, zd - d on one tape row) at the chunk's first and last row, and in its middle."""
    import os
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    os.environ['ZKA_TOM_W'] = '16'          # small fixed-base tables beside the session's engines; c does not depend on them
    try:
        L = ZkaLib(g.LIB_WAR if war else g.LIB)
    finally:
        os.environ.pop('ZKA_TOM_W', None)
    cpu = None if war else _cpu_port()     # oracle/cpu is a tomEdwards256 build; war256 rows go to the Python oracle
    B, sec = 4096, 80
    bt = Batch(L, B, 89, sec=sec, ring_size=256)
    try:
        pa, pb = shifted(bt.row0, 'zd', D, sec), shifted(bt.row0, 'zd', -D, sec)
        for ia, ib in ((0, B - 1), (2047, 2048)):
            run_case(bt, pair(bt, pa, pb, ia, ib), chunk=B, cpu=cpu, python=war)
        assert 12 <= L.stat('agg_c') <= 16, L.stat('agg_c')
        all_share_one_tape(bt, chunk=B)
    finally:
        bt.close()
        L.close()


# ------------------------------------------------------------------------------------------------ the weights
# A model of AggWeightTask (zk_verify_agg.cuh), input by input.  `omit` drops inputs from it, as a forger who assumed a
# weaker derivation would: 'msg', 'tags', 'chal', 'header', 'tape', 'reps', 'gk'.  The device stores digests as
# big-endian words and hashes them as they lie in memory: little-endian bytes of each word.
def _lew(digest):
    return b''.join(digest[i:i + 4][::-1] for i in range(0, 32, 4))


def _sha(b):
    import hashlib
    return hashlib.sha256(b).digest()


def model_weights(row, ring_index, msg, proof, tape_row, ring_size, sec=SEC, K=SEC, omit=()):
    """(wG, wW, wN) of row `row` of a call, as integers (the factors the aggregate applies)."""
    import struct
    n = VT.ceil_log2(ring_size)
    off, offs, tags = flat.HEAD_LEN, [], [0, 0, 0]
    for i in range(sec):
        offs.append(off)
        if proof[off]:
            tags[i >> 5] |= 1 << (i & 31)
        off += flat.REP1_LEN if proof[off] else flat.REP0_LEN
    gk_off, plen = off, len(proof)
    perm = list(range(sec))
    ib = tape_row[32 * (2 * n + 1):]
    for i in range(sec - 2):
        r = ib[i] if ib[i] < sec - i else 0
        perm[i], perm[r + i] = perm[r + i], perm[i]
    chal = _sha(proof[2 * flat.NP:2 * flat.NP + 2 * flat.WP]
                + b''.join(proof[o + 1:o + 1 + flat.NP + 2 * flat.WP] for o in offs))
    tape_len = VT.verify_tape_len(ring_size, K)
    pieces = [(tape_row[lo:min(lo + 2048, tape_len)], 'tape') for lo in range(0, tape_len, 2048)]
    for i in perm[:K]:
        hi = offs[i] + (flat.REP1_LEN if tags[i >> 5] >> (i & 31) & 1 else flat.REP0_LEN)
        pieces.append((proof[offs[i]:min(hi, plen)], 'reps'))
    pieces.append((proof[gk_off:plen], 'gk'))
    parts = [struct.pack('<4I', 0x5741475a, row, ring_index, plen),
             b'' if 'msg' in omit else msg,
             b'' if 'tags' in omit else struct.pack('<3I', *tags),
             b'' if 'chal' in omit else _lew(chal),
             b'' if 'header' in omit else proof[:flat.HEAD_LEN]]
    parts += [_lew(_sha(p)) for p, kind in pieces if kind not in omit]
    d = _lew(_sha(b''.join(parts)))
    out = []
    for j in range(3):
        o = _sha(d + struct.pack('<I', j))
        w = [int.from_bytes(o[4 * k:4 * k + 4], 'big') for k in range(4)]
        out.append((w[3] | 1) | w[2] << 32 | w[1] << 64 | w[0] << 96)
    return out


PROOF_PARTS = ('msg', 'tags', 'chal', 'header', 'reps', 'gk')
INDEX_ONLY = PROOF_PARTS + ('tape',)


def check_model_is_the_library(L, seed=93):
    """The model is the library's derivation bit for bit.  The ring is a verifier input that no weight covers: two
    ring entries solved against the model's GK weights make the GK residuals of two valid rows cancel in the weighted
    sum, and the library then counts the chunk as decided by the aggregate.  So the forgeries below, built against
    weaker models, are tried against the real weights."""
    from oracle.curves import hash_points
    bt = Batch(L, 2, seed)
    try:
        grp = bt.po.ProofGroup.c
        q = grp.order
        n = VT.ceil_log2(bt.N)
        rows = [bt.proofs[b, :bt.plen[b]].tobytes() for b in range(2)]
        coef = []                                   # rho_b * pix_b(i) for ring entries 1 and 2
        for b in range(2):
            prf = flat.de_proof(rows[b], SEC)
            gk = prf.membershipProof
            x = hash_points(gk.cl + gk.ca + gk.cb + gk.cd)

            def pix(i):
                v = 1
                for j in range(n):
                    v = v * (gk.f[j].k if i >> j & 1 else x - gk.f[j].k) % q
                return v
            vec = [v % q for v in bt.ring_ints] + [bt.ring_ints[0] % q] * ((1 << n) - bt.N)
            total = sum(vec[i] * pix(i) for i in range(1 << n)) % q
            rels = relations(bt.po, bt.wl.msg_hash[b].tobytes(), bt.ring_ints, rows[b], bt.vt[b].tobytes())
            rho = rho_of(rels, grp, -total)
            wG = model_weights(b, 0, bt.wl.msg_hash[b].tobytes(), rows[b], bt.vt[b].tobytes(), bt.N)[0]
            coef.append((wG * rho * pix(1) % q, wG * rho * pix(2) % q))
        d2 = -(coef[0][0] + coef[1][0]) * pow(coef[0][1] + coef[1][1], -1, q) % q
        ring = bt.wl.ring.copy()
        for i, d in ((1, 1), (2, d2)):
            ring[i] = np.frombuffer(((bt.ring_ints[i] + d) % q).to_bytes(32, 'big'), np.uint8)
        ring_ints = [int.from_bytes(r.tobytes(), 'big') for r in ring]
        for b in range(2):
            assert common.oracle_verdict(bt.po, bt.wl.msg_hash[b].tobytes(), ring_ints, rows[b], bt.vt[b].tobytes(), bt.N,
                                         SEC) is False

        def call(ok, st):
            L.verify_batch(bt.P, 2, bt.wl.msg_hash, ring, bt.N, bt.proofs, bt.proofs.shape[1], bt.plen, bt.vt, bt.vt.shape[1],
                           ok, st)
        ok, st, dp, df, ok2, st2, _ = verify_both(L, call, 2)
        assert list(ok2) == [0, 0] and not st2.any()                    # the per-proof path: the reference's verdicts
        assert (dp, df) == (1, 0) and list(ok) == [1, 1], (dp, df, list(ok))   # the weighted sum cancels: exact model
    finally:
        bt.close()


def check_weaker_weights(L, B=6, seed=95):
    """Forgers who know a weaker derivation than the library's: each builds a pair (or a row) that cancels under its
    model, and the library must reject it.  A library whose weights left out the input the forger left out would
    accept it (check_model_is_the_library shows the model is exact)."""
    bt = Batch(L, B, seed)
    try:
        msg = bt.wl.msg_hash[0].tobytes()
        t = bt.vt[0].tobytes()
        ia, ib = 1, B - 2
        q_t, q_n = flat.PROOF_GROUP.order, p256.order

        def w(i, p, omit, j, tape=t):
            return model_weights(i, 0, msg, p, tape, bt.N, omit=omit)[j]

        # shared tape row, responses shifted by dA and dB with wA dA + wB dB = 0: the forger's model leaves out the part
        # of the proof that holds the response (or every input but the row index)
        for field, j, q, omit in (('zd', 0, q_t, ('gk',)), ('zd', 0, q_t, INDEX_ONLY), ('beta2', 1, q_t, ('reps',)),
                                  ('beta1', 2, q_n, ('reps',)), ('za', 0, q_t, PROOF_PARTS)):
            pa = shifted(bt.row0, field, D)
            db = -w(ia, pa, omit, j) * D * pow(w(ib, bt.row0, omit, j), -1, q) % q
            pb = shifted(bt.row0, field, db)
            assert w(ib, pb, omit, j) == w(ib, bt.row0, omit, j)       # blind to the shift, as the forger assumed
            run_case(bt, pair(bt, pa, pb, ia, ib))
        # comS1 (multiN, held by every 0-bit relA with the same randomizers on a shared tape row) + X and + Y, with
        # wA X + wB Y = O for a model without the header
        X = bt.po.NistGroup.g.mul(p256.new_scalar(D))

        def with_coms1(k):
            prf = flat.de_proof(bt.row0, SEC)
            prf.comS1 = prf.comS1.add(X.mul(p256.new_scalar(k)))
            return flat.ser_proof(prf)
        pa = with_coms1(1)
        kb = -w(ia, pa, ('header',), 2) * pow(w(ib, bt.row0, ('header',), 2), -1, q_n) % q_n
        run_case(bt, pair(bt, pa, with_coms1(kb), ia, ib))
        # distinct tape rows and a tape-aware forger whose model has no proof binding at all (family 3 with weights)
        tb = bt.vt[B - 1].tobytes()
        for fa, fb, j, q in (('zd', 'zd', 0, q_t), ('beta1', 'z2', 2, q_n)):
            pa = shifted(bt.row0, fa, D)
            ratio = w(ia, pa, PROOF_PARTS, j) * pow(w(ib, bt.row0, PROOF_PARTS, j, tb), -1, q) % q
            db = cancel_shift(bt, fa, D * ratio % q, t, fb, tb)
            run_case(bt, pair(bt, pa, shifted(bt.row0, fb, db), ia, ib, t, tb))
        # one row, GK against multiW (family 4) with a model that knows neither the GK block nor the repetitions
        omit = ('gk', 'reps')
        p1 = shifted(bt.row0, 'zd', D)
        ratio = w(ia, p1, omit, 0) * pow(w(ia, p1, omit, 1), -1, q_t) % q_t
        d2 = cancel_shift(bt, 'zd', D * ratio % q_t, t, 'beta2', t)
        run_case(bt, {ia: (shifted(p1, 'beta2', d2), t)})
    finally:
        bt.close()


def test_weight_model_is_the_library_hostsim(sim):
    check_model_is_the_library(sim)


def test_forgers_with_weaker_weights_hostsim(sim):
    check_weaker_weights(sim)


@pytest.mark.gpu
def test_weights_on_gpu(gpu):
    check_model_is_the_library(gpu)
    check_weaker_weights(gpu)
