"""Parity tests proper: the sm_90a library through the C ABI vs the oracle (run on an H100)."""
import numpy as np
import pytest

import common
from zkp_ecdsa_b200 import synth

pytestmark = pytest.mark.gpu


def test_field_ops(gpu_engine):
    common.check_field_ops(gpu_engine.lib, count=200)


def test_hash80(gpu_engine):
    common.check_hash(gpu_engine.lib)


def test_p256_mul(gpu_engine):
    common.check_p256_mul(gpu_engine.lib, count=12)
    common.check_noncanonical_p256(gpu_engine.lib)


def test_params_and_commit(gpu_engine):
    P, po = common.make_params(gpu_engine.lib, seed=5)
    common.check_tom_commit(gpu_engine.lib, P, po, count=12)
    gpu_engine.lib.params_destroy(P)


def test_prove_bit_exact_small_ring(gpu_engine):
    common.check_prove_parity(gpu_engine.lib, B=2, N=6, seed=3)


def test_prove_bit_exact_ring_256(gpu_engine):
    common.check_prove_parity(gpu_engine.lib, B=2, N=256, seed=8)


def test_prove_bit_exact_sec_level_16(gpu_engine):
    common.check_prove_parity(gpu_engine.lib, B=5, N=17, seed=4, sec_level=16)


def test_prove_batch_properties_config2(gpu_engine):
    """BASELINE config 2 shape (batch 1024, ring 8): size-independent properties."""
    L = gpu_engine.lib
    P, po = common.make_params(L, seed=21)
    B, N = 1024, 8
    wl = synth.Workload(B=B, N=N, seed=21)
    tape = synth.random_tape(B, L.prove_tape_len(N), seed=22)
    proofs, plen, status = common.run_prove(L, P, wl, tape)
    assert (status == 0).all()
    from oracle import flat
    # lengths follow the layout formula; zero bits are binomial(80, 1/2)
    zs = (plen.astype(np.int64) - flat.proof_len(0, 3)) // (flat.REP0_LEN - flat.REP1_LEN)
    assert ((plen == [flat.proof_len(int(z), 3) for z in zs])).all()
    assert 30 < zs.mean() < 50
    # determinism: same inputs -> same bytes; different tape -> different proof
    proofs2, plen2, _ = common.run_prove(L, P, wl, tape)
    assert (plen == plen2).all() and (proofs == proofs2).all()
    # spot-check three proofs bit-exactly against the oracle
    for b in (0, 511, 1023):
        pr, _ = common.oracle_proof(po, wl, tape, b)
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr)
    L.params_destroy(P)


def test_error_statuses(gpu_engine):
    L = gpu_engine.lib
    P, po = common.make_params(L, seed=31)
    wl = synth.Workload(B=4, N=8, seed=31)
    tape = synth.random_tape(4, L.prove_tape_len(8), seed=32)
    wl.pk[1, 40] ^= 1                      # not on the curve -> 'invalid public key'
    wl.which[2] = 8                        # outside the ring
    tape[3, 32 * 3:32 * 3 + 4] = 255       # alpha_0 >= n -> tape range
    _, _, status = common.run_prove(L, P, wl, tape)
    assert list(status) == [0, 1, 6, 5]
    L.params_destroy(P)


def test_verify_decisions_match_oracle(gpu_engine):
    common.check_verify_parity(gpu_engine.lib, N=6, seed=3, tampers=32)


def test_verify_ring_256(gpu_engine):
    common.check_verify_parity(gpu_engine.lib, N=256, seed=12, tampers=8)


def test_prove_verify_roundtrip_batch(gpu_engine):
    """encode -> verify round trip at batch 512, ring 1024 (size-independent property)."""
    from zkp_ecdsa_b200 import verify_tape as VT
    L = gpu_engine.lib
    P, po = common.make_params(L, seed=41)
    B, N = 512, 1024
    wl = synth.Workload(B=B, N=N, seed=41)
    tape = synth.random_tape(B, L.prove_tape_len(N), seed=42)
    proofs, plen, status = common.run_prove(L, P, wl, tape)
    assert (status == 0).all()
    vt = VT.random_verify_tape(B, L.verify_tape_len(N), N, seed=43)
    ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
    assert (st == 0).all() and (ok == 1).all()
    # swap two messages: exactly those two verifications must fail
    msg = wl.msg_hash.copy()
    msg[[3, 4]] = msg[[4, 3]]
    ok, st = common.run_verify(L, P, msg, wl.ring, proofs, plen, vt)
    assert (st == 0).all() and list(np.nonzero(ok == 0)[0]) == [3, 4]
    L.params_destroy(P)


def test_edge_cases_on_gpu(gpu_engine):
    import test_edge_cases as E
    L = gpu_engine.lib
    E.test_ring_of_two(L)
    E.test_ragged_ring_signer_last(L)
    E.test_zero_message_hash(L)
    E.test_zero_r_and_zero_s(L)
    E.test_key_to_int(L)


def test_alternate_code_paths_on_gpu():
    """Paths the default engine does not take: ragged / small table windows, and a ring above 1024
    entries (Groth-Kohlweiss block sums)."""
    import os
    from zkp_ecdsa_b200 import api
    os.environ.update(ZKA_TOM_W='14', ZKA_P256_HW='11')
    try:
        eng = api.Engine(device=0)
    finally:
        for k in ('ZKA_TOM_W', 'ZKA_P256_HW'):
            os.environ.pop(k, None)
    try:
        common.check_prove_parity(eng.lib, B=3, N=6, sec_level=80, seed=41)
        common.check_prove_parity(eng.lib, B=1, N=2100, sec_level=20, seed=42)
        common.check_verify_parity(eng.lib, N=2100, sec_level=20, seed=43, tampers=4)
    finally:
        eng.close()


def test_edge_tapes_on_gpu(gpu_engine, gpu_engine_war):
    """Edge scalars in every prover and verifier tape draw (synth.edge_tape, verify_tape.edge_verify_tape) at SecLevel
    80: proofs against the Python oracle, verdicts against oracle/cpu, the aggregate MSM at its default window and
    c = 4, 9, 13, 16 — with the default table windows, with 14 / 11-bit windows, and on the war256 build."""
    import os
    from functools import partial
    from zkp_ecdsa_b200 import api, verify_tape as VT
    import test_verify_aggregate as tva
    e80 = partial(synth.edge_tape, sec_level=80)
    os.environ.update(ZKA_TOM_W='14', ZKA_P256_HW='11')
    try:
        narrow = api.Engine(device=0)
    finally:
        for k in ('ZKA_TOM_W', 'ZKA_P256_HW'):
            os.environ.pop(k, None)
    try:
        for L in (gpu_engine.lib, narrow.lib):
            common.check_prove_parity(L, B=2, N=6, seed=301, make_tape=e80)
            common.check_verify_samples(L, 20, N=5, seed=302, tampers=4, oracle=_cpu_port(), make_tape=e80,
                                        make_vtape=VT.edge_verify_tape)
            # the chunk of test_edge_cases.test_edge_tapes (3 proofs the reference accepts: some edge prover tapes give a
            # proof that the reference's own verifier rejects, and then so does this library)
            tva.check_aggregate(L, B=3, N=6, seed=203, cs=(0, 4, 9, 13, 16), ks=(33,), make_tape=e80,
                                make_vtape=VT.edge_verify_tape)
    finally:
        narrow.close()
    L = gpu_engine_war.lib
    common.check_prove_parity(L, B=2, N=6, seed=311, make_tape=e80)
    common.check_verify_parity(L, N=6, seed=312, tampers=4, make_tape=e80, make_vtape=VT.edge_verify_tape)
    tva.check_aggregate(L, B=3, N=6, seed=213, cs=(0, 4, 9, 13, 16), ks=(33,), make_tape=e80,
                        make_vtape=VT.edge_verify_tape)


# ---------------------------------------------------------------------------------- round 2
def _cpu_port():
    """oracle/cpu (C++ restatement of the reference algorithms): the fast checker for big shapes."""
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    assert __import__('os').path.exists(g.ORACLE_CPU), 'oracle/_ref/libzkattest_cpu.so missing: run build()'
    return ZkaLib(g.ORACLE_CPU)


def _spot_check(cpu, po_rnd, wl, tape, proofs, plen, spots, sec=80, python_spot=None):
    """proofs[b] == oracle proof for b in spots (C++ port; one of them also against the Python oracle)."""
    from oracle import flat
    hn, hp = cpu.params_generate(po_rnd)
    Pc = cpu.params_create(hn, hp, sec)
    idx = np.array(spots)
    sub = synth.Workload.__new__(synth.Workload)
    sub.B, sub.N = len(spots), wl.N
    sub.msg_hash, sub.sig, sub.pk, sub.which, sub.ring = (np.ascontiguousarray(wl.msg_hash[idx]), np.ascontiguousarray(wl.sig[idx]),
                                                            np.ascontiguousarray(wl.pk[idx]), np.ascontiguousarray(wl.which[idx]), wl.ring)
    ref, rlen, rst = common.run_prove(cpu, Pc, sub, np.ascontiguousarray(tape[idx]), sec)
    assert not rst.any()
    for k, b in enumerate(spots):
        assert plen[b] == rlen[k] and proofs[b, :plen[b]].tobytes() == ref[k, :rlen[k]].tobytes(), f'proof {b} differs from oracle/cpu'
    if python_spot is not None:
        from oracle import zkattest as OZ
        from oracle.big import Tape
        po = OZ.generate_params_list(Tape(po_rnd), sec)
        pr, _ = common.oracle_proof(po, wl, tape, python_spot)
        assert proofs[python_spot, :plen[python_spot]].tobytes() == flat.ser_proof(pr)
    cpu.params_destroy(Pc)


def test_config3_shape_spot_proofs_bit_exact(gpu_engine):
    """BASELINE configs[3] shape per GPU: 8192 proofs, ring N = 1024, SecLevel 80.  Three spot proofs are compared
    byte for byte with the oracle (C++ port; proof 0 also with the Python oracle), all lengths with the layout law."""
    from oracle import flat
    L = gpu_engine.lib
    rnd = synth.params_rnd(51)
    P, _ = common.make_params(L, seed=51)
    B, N = 8192, 1024
    wl = synth.Workload(B=B, N=N, seed=51)
    tape = synth.random_tape(B, L.prove_tape_len(N), seed=52)
    proofs, plen, status = common.run_prove(L, P, wl, tape)
    assert (status == 0).all()
    zs = (plen.astype(np.int64) - flat.proof_len(0, 10)) // (flat.REP0_LEN - flat.REP1_LEN)
    assert (plen == [flat.proof_len(int(z), 10) for z in zs]).all() and 38 < zs.mean() < 42
    _spot_check(_cpu_port(), rnd, wl, tape, proofs, plen, [0, 4097, 8191], python_spot=0)
    L.params_destroy(P)


def test_host_pipeline_chunks_and_lanes_bit_exact(gpu_engine):
    """B = 1024 with host buffers through >= 4 chunks of the three-stream pipeline, on 1, 2 and 3 lanes, must equal
    the single-chunk device-pointer result and the oracle; the same for the verifier."""
    import torch
    from zkp_ecdsa_b200 import verify_tape as VT
    L = gpu_engine.lib
    rnd = synth.params_rnd(61)
    P, _ = common.make_params(L, seed=61)
    B, N = 1024, 8
    wl = synth.Workload(B=B, N=N, seed=61)
    ts, ps, vts = L.prove_tape_len(N), L.proof_max_len(N), L.verify_tape_len(N)
    tape = synth.random_tape(B, ts, seed=62)
    vt = VT.random_verify_tape(B, vts, N, 80, seed=63)
    cfg0 = L.config()
    dev = torch.device('cuda', 0)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)   # noqa: E731
    d = [t(wl.msg_hash), t(wl.sig), t(wl.pk), t(wl.which.view(np.uint8)), t(wl.ring), t(tape), t(vt)]
    pd = torch.zeros((B, ps), dtype=torch.uint8, device=dev)
    ld = torch.zeros(B, dtype=torch.int32, device=dev)
    sd = torch.zeros(B, dtype=torch.int32, device=dev)
    okd = torch.zeros(B, dtype=torch.uint8, device=dev)
    try:
        L.set_option('lanes', 1)
        L.set_option('chunk', 8192)
        L.prove_batch(P, B, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), N, d[5].data_ptr(),
                      ts, pd.data_ptr(), ps, ld.data_ptr(), sd.data_ptr())
        ref_p, ref_l = pd.cpu().numpy(), ld.cpu().numpy().astype(np.uint32)
        assert not sd.cpu().numpy().any()
        _spot_check(_cpu_port(), rnd, wl, tape, ref_p, ref_l, [0, 300, 1023])
        L.set_option('host_chunk', 256)
        for lanes in (1, 2, 3):
            L.set_option('lanes', lanes)
            proofs, plen, status = common.run_prove(L, P, wl, tape)
            assert not status.any() and (plen == ref_l).all(), lanes
            for b in range(B):
                assert (proofs[b, :plen[b]] == ref_p[b, :plen[b]]).all(), (lanes, b)
            # verifier: host buffers, 256-proof chunks, `lanes` lanes; then one tampered message
            L.set_option('chunk', 256)
            ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
            assert (ok == 1).all() and not st.any(), lanes
            msg = wl.msg_hash.copy()
            msg[777, 3] ^= 8
            ok, st = common.run_verify(L, P, msg, wl.ring, proofs, plen, vt)
            assert list(np.nonzero(ok == 0)[0]) == [777] and not st.any()
            L.set_option('chunk', 8192)
        # device-pointer verification of the device-resident proofs
        L.verify_batch(P, B, d[0].data_ptr(), d[4].data_ptr(), N, pd.data_ptr(), ps, ld.data_ptr(), d[6].data_ptr(), vts,
                       okd.data_ptr(), sd.data_ptr())
        assert bool((okd == 1).all().item()) and not sd.cpu().numpy().any()
    finally:
        L.set_option('lanes', cfg0['lanes'])
        L.set_option('chunk', cfg0['chunk'])
        L.set_option('host_chunk', 4096)
    L.params_destroy(P)


def test_wild_index_and_error_rows_on_gpu(gpu_engine):
    """`which` = 0xFFFFFFFF must not fault (the GK tasks read a clamped copy) and failed proofs leave as zero rows."""
    L = gpu_engine.lib
    P, po = common.make_params(L, seed=71)
    wl = synth.Workload(B=4, N=8, seed=71)
    wl.which[1] = 0xFFFFFFFF
    wl.which[3] = 1 << 20
    wl.pk[2, 10] ^= 4
    tape = synth.random_tape(4, L.prove_tape_len(8), seed=72)
    proofs, plen, status = common.run_prove(L, P, wl, tape)
    assert list(status) == [0, 6, 1, 6]
    assert plen[0] > 0 and not plen[1:].any() and not proofs[1:].any()
    from oracle import flat
    pr, _ = common.oracle_proof(po, wl, tape, 0)
    assert proofs[0, :plen[0]].tobytes() == flat.ser_proof(pr)
    # the context is still healthy
    common.check_prove_parity(L, B=1, N=6, seed=73, sec_level=16)
    L.params_destroy(P)


def test_verify_sample_count_on_gpu(gpu_engine):
    """zka_verify_batch_ex: 5, 33 and all 80 repetitions sampled (80 = four MSM segments per proof); verdicts on valid
    and tampered proofs equal oracle/cpu's under identical randomness."""
    cpu = _cpu_port()
    for K in (5, 33, 80):
        common.check_verify_samples(gpu_engine.lib, K, N=5, seed=25, sec_level=80, tampers=6, oracle=cpu)
    common.check_verify_samples(gpu_engine.lib, 7, N=4, seed=26, sec_level=20, tampers=2, oracle='python')


@pytest.mark.gpu
def test_prove_few_distinct_keys_wide_key_tables_on_gpu(gpu_engine):
    """256 proofs of 2 / 40 signers: the per-key tables use 8-bit / 7-bit windows (device-chosen) instead of 5."""
    common.check_prove_few_keys(gpu_engine.lib, B=256, N=64, signers=2, seed=43, sec_level=80, spots=(0, 255))
    common.check_prove_few_keys(gpu_engine.lib, B=256, N=64, signers=40, seed=44, sec_level=16, spots=(5, 130, 255))
