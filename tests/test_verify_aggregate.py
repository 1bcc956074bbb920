"""Chunk-wide aggregate check of the verifier (zk_verify_agg.cuh): a valid chunk is accepted by ONE wide-window MSM per
group; a chunk holding a wrong proof falls back to the per-proof evaluation and gives exactly its verdicts."""
import numpy as np
import pytest

import common
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT


def _batch(L, B, N, seed, sec_level=80, make_tape=synth.random_tape, make_vtape=VT.random_verify_tape):
    P, po = common.make_params(L, seed, sec_level)
    wl = synth.Workload(B=B, N=N, seed=seed)
    tape = make_tape(B, L.prove_tape_len(N, sec_level), seed=seed + 100)
    proofs, plen, status = common.run_prove(L, P, wl, tape, sec_level)
    assert (status == 0).all()
    vt = make_vtape(B, L.verify_tape_len(N, sec_level), N, sec_level, seed=seed + 7)
    return P, wl, proofs, plen, vt


def check_aggregate(L, B=5, N=6, seed=31, cs=(0, 4, 7, 11), ks=(33,), make_tape=synth.random_tape,
                    make_vtape=VT.random_verify_tape):
    """make_tape / make_vtape: the prover and verifier tape makers (random, or edge scalars in every draw)."""
    P, wl, proofs, plen, vt = _batch(L, B, N, seed, make_tape=make_tape, make_vtape=make_vtape)
    try:
        for c in cs:
            if c:
                L.set_option('agg_c', c)
            p0, f0 = L.stat('agg_pass'), L.stat('agg_fail')
            ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
            assert list(ok) == [1] * B and not st.any(), (c, ok, st)
            assert L.stat('agg_pass') > p0 and L.stat('agg_fail') == f0, c      # decided by the aggregate
        # other sample counts (verifyExp's secparam): 33 and all 80 repetitions = 2 / 4 MSM segments per proof
        for K in ks:
            vtk = make_vtape(B, L.verify_tape_len_ex(N, 80, K), N, 80, seed=seed + K)
            okk = np.zeros(B, np.uint8)
            stk = np.zeros(B, np.int32)
            p0, f0 = L.stat('agg_pass'), L.stat('agg_fail')
            L.verify_batch_ex(P, B, wl.msg_hash, wl.ring, N, proofs, proofs.shape[1], plen, vtk, vtk.shape[1], okk, stk, K)
            assert list(okk) == [1] * B and not stk.any(), (K, okk, stk)
            assert L.stat('agg_pass') > p0 and L.stat('agg_fail') == f0, K
        # one wrong proof (a flipped bit in the last GK response scalar, which every verification reads): the chunk
        # goes to the per-proof path
        bad = proofs.copy()
        bad[2, plen[2] - 1] ^= 1
        p0, f0 = L.stat('agg_pass'), L.stat('agg_fail')
        ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, bad, plen, vt)
        assert L.stat('agg_fail') > f0 and L.stat('agg_pass') == p0
        L.set_option('agg', 1)                                                   # aggregate off: the reference verdicts
        ok2, st2 = common.run_verify(L, P, wl.msg_hash, wl.ring, bad, plen, vt)
        okv, stv = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
        assert L.stat('agg_fail') == f0 + (L.stat('agg_fail') - f0) and list(okv) == [1] * B and not stv.any()
        L.set_option('agg', 2)
        assert (ok == ok2).all() and (st == st2).all()
        assert ok[2] == 0 and list(np.delete(ok, 2)) == [1] * (B - 1), ok
        # a malformed row (truncated) keeps its own status and sends the chunk to the per-proof path too
        plen2 = plen.copy()
        plen2[1] -= 3
        ok3, st3 = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen2, vt)
        assert ok3[1] == 0 and st3[1] != 0 and list(np.delete(ok3, 1)) == [1] * (B - 1)
    finally:
        L.set_option('agg', 2)
        L.set_option('agg_c', 6)
        L.params_destroy(P)


def test_aggregate_check_hostsim(hostsim):
    check_aggregate(hostsim)


@pytest.mark.gpu
def test_aggregate_check_on_gpu(gpu_engine):
    check_aggregate(gpu_engine.lib, B=40, N=17, seed=33, cs=(0, 9, 13), ks=(33, 80))


def check_small_order_components(L, B=6, N=5, seed=91, sec_level=20, trials=8):
    """tomEdwards256 has cofactor 4 and deserializePoint only checks the curve equation.  Proofs whose A_1 points of pi_x
    carry the point of order 2 (added BEFORE the Fiat-Shamir hash, so everything else is consistent) are accepted by the
    reference exactly when an even number of the affected relations got an odd randomizer.  Two rejected proofs of one
    chunk would cancel in the chunk-wide sum — the torsion guard must send such a chunk to the per-proof path, whose
    verdicts are the oracle's under the same tape."""
    from oracle import commit as OC
    from oracle import exp as OE
    from oracle.curves import hash_points, tomEdwards256 as tom
    from oracle.big import rnd
    assert L.group == 'tomEdwards256'
    P, po = common.make_params(L, seed, sec_level)
    T2 = tom.deserialize_point(b'\x04' + (0).to_bytes(33, 'big') + (tom.p - 1).to_bytes(33, 'big'))     # (0, -1): order 2
    assert T2.add(T2).is_identity() and not T2.is_identity()

    def prove_equality_t2(params, x, C1, C2, tape):      # equality.ts:60-78 with A_1 + T2
        k = rnd(params.c.order, tape)
        A1 = params.commit(k, tape)
        A2 = params.commit(k, tape)
        A1p = A1.p.add(T2)
        c = hash_points([C1.p, C2.p, A1p, A2.p])
        cc, xx, kk = params.c.new_scalar(c), params.c.new_scalar(x), params.c.new_scalar(k)
        return OC.EqualityProof(A1p, A2.p, kk.sub(cc.mul(xx)), A1.r.sub(cc.mul(C1.r)), A2.r.sub(cc.mul(C2.r)))
    wl = synth.Workload(B=B, N=N, seed=seed)
    tape = synth.random_tape(B, L.prove_tape_len(N, sec_level), seed=seed + 100)
    orig = OE.prove_equality
    OE.prove_equality = prove_equality_t2
    try:
        rows = [common.flat.ser_proof(common.oracle_proof(po, wl, tape, b)[0]) for b in range(B)]
    finally:
        OE.prove_equality = orig
    ps = L.proof_max_len(N, sec_level)
    proofs = np.zeros((B, ps), np.uint8)
    plen = np.zeros(B, np.uint32)
    for b, r in enumerate(rows):
        proofs[b, :len(r)] = np.frombuffer(r, np.uint8)
        plen[b] = len(r)
    vts = L.verify_tape_len(N, sec_level)
    ring_ints = wl.ring_ints()
    dangerous = 0
    try:
        for t in range(trials):
            vt = VT.random_verify_tape(B, vts, N, sec_level, seed=seed + 7 + t)
            exp = [common.oracle_verdict(po, wl.msg_hash[b].tobytes(), ring_ints, rows[b], vt[b].tobytes(), N, sec_level) for b in range(B)]
            assert all(e in (True, False) for e in exp), exp
            p0 = L.stat('agg_pass')
            ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
            assert not st.any() and [bool(v) for v in ok] == exp, (t, list(ok), exp)
            rejected = exp.count(False)
            if rejected:
                assert L.stat('agg_pass') == p0          # never decided by the aggregate
            if rejected >= 2 and rejected % 2 == 0:
                dangerous += 1                           # the components would have cancelled in the sum
        assert dangerous >= 1, 'no trial had an even number (>= 2) of rejected proofs: pick other seeds'
    finally:
        L.params_destroy(P)


def test_small_order_components_hostsim(hostsim):
    check_small_order_components(hostsim)


@pytest.mark.gpu
def test_small_order_components_on_gpu(gpu_engine):
    check_small_order_components(gpu_engine.lib)      # same inputs as on the host simulator (3 of the 8 trials cancel)
