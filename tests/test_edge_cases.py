"""Edge cases of the path (empty/ragged/degenerate inputs) — host simulator here, GPU in test_gpu_parity."""
import numpy as np
import pytest

import common
from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from zkp_ecdsa_b200 import synth, verify_tape as VT


def _roundtrip(L, N, seed, sec=16, mutate=None, which_last=False):
    P, po = common.make_params(L, seed, sec)
    wl = synth.Workload(B=2, N=N, seed=seed)
    if which_last:   # signer in the last ring slot
        j = int(wl.which[0])
        wl.ring[[j, N - 1]] = wl.ring[[N - 1, j]]
        if int(wl.which[1]) == N - 1:
            wl.which[1] = j
        wl.which[0] = N - 1
    if mutate:
        mutate(wl)
    tape = synth.random_tape(2, L.prove_tape_len(N, sec), seed=seed + 1)
    proofs, plen, status = common.run_prove(L, P, wl, tape, sec)
    exp_status = []
    for b in range(2):
        try:
            pr, _ = common.oracle_proof(po, wl, tape, b)
            assert status[b] == 0, (b, status)
            assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), b
            exp_status.append(0)
        except ValueError:
            assert status[b] != 0, (b, 'oracle throws, GPU status 0')
            exp_status.append(1)
    if sec >= 20:
        vt = VT.random_verify_tape(2, L.verify_tape_len(N, sec), N, sec, seed=seed + 2)
        ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
        for b in range(2):
            if exp_status[b] == 0:
                want = common.oracle_verdict(po, wl.msg_hash[b].tobytes(), wl.ring_ints(), proofs[b, :plen[b]].tobytes(),
                                             vt[b].tobytes(), N, sec)
                got = 'err' if st[b] else bool(ok[b])
                assert got == want, (b, got, want)
    L.params_destroy(P)
    return status


def test_ring_of_two(hostsim):
    _roundtrip(hostsim, N=2, seed=51, sec=20)


def test_ragged_ring_signer_last(hostsim):
    _roundtrip(hostsim, N=5, seed=52, sec=20, which_last=True)     # padded 5 -> 8 with ring[0] (gk.ts:80-83)


def test_zero_message_hash(hostsim):
    # z = 0 -> z1 = 0 -> Q is the identity (zkpAttestList.ts:134-136): T1 = R*z + O
    def mut(wl):
        wl.msg_hash[0] = 0
    st = _roundtrip(hostsim, N=4, seed=53, sec=20, mutate=mut)
    assert list(st) == [0, 0]          # the prover does not check the signature; the proof is well formed


def test_zero_r_and_zero_s(hostsim):
    def mut(wl):
        wl.sig[0, :32] = 0             # r = 0: rinv = 0 -> "Points don't add up!" (pointAdd.ts:105)
        wl.sig[1, 32:] = 0             # s = 0: R is the identity -> 'T[i] is at infinity' (exp.ts:151)
    st = _roundtrip(hostsim, N=4, seed=54, sec=16, mutate=mut)
    assert st[0] == 4 and st[1] == 2


def test_ring_size_one_is_rejected(hostsim):
    # hashPoints([]) throws in the reference (group.ts:223 reduce of an empty array): argument error here
    from zkp_ecdsa_b200.capi import ZkaError
    P, _ = common.make_params(hostsim, 55, 16)
    wl = synth.Workload(B=1, N=2, seed=55)
    wl.ring = wl.ring[:1].copy()
    wl.N = 1
    tape = synth.random_tape(1, hostsim.prove_tape_len(2, 16), seed=1)
    with pytest.raises(ZkaError):
        common.run_prove(hostsim, P, wl, tape, 16)
    hostsim.params_destroy(P)


def test_verify_needs_20_repetitions(hostsim):
    # verifyExp throws 'security level not achieved' when SecLevel < 20 (exp.ts:243-245)
    from zkp_ecdsa_b200.capi import ZkaError
    P, po = common.make_params(hostsim, 56, 16)
    wl = synth.Workload(B=1, N=4, seed=56)
    tape = synth.random_tape(1, hostsim.prove_tape_len(4, 16), seed=2)
    proofs, plen, status = common.run_prove(hostsim, P, wl, tape, 16)
    vt = VT.random_verify_tape(1, hostsim.verify_tape_len(4, 16), 4, 80, seed=3)
    with pytest.raises(ZkaError):
        common.run_verify(hostsim, P, wl.msg_hash, wl.ring, proofs, plen, vt)
    hostsim.params_destroy(P)


def test_key_to_int(hostsim):
    wl = synth.Workload(B=3, N=4, seed=57)
    pk = wl.pk.copy()
    pk[2, 10] ^= 1
    x, st = hostsim.key_to_int(pk)
    assert list(st) == [0, 0, 1]
    for b in range(2):
        assert int.from_bytes(x[b].tobytes(), 'big') == OZ.key_to_int(wl.pk[b].tobytes())


def check_edge_tapes(L, seed, sec_prove=16, sec_verify=20, cs=(0, 4, 9, 13, 16)):
    """Every 32-byte draw of the prover and verifier tapes an edge scalar (1, m-1, the top 2^-32 of the range, single
    bits, windows all 2^(w-1) or 2^(w-1)+1): commitment scalars, blinders, k's, GK draws and the verifier's MSM
    randomizers go through the table lookups, the per-proof MSMs and the aggregate MSM at every window width `cs`."""
    from functools import partial
    edge = lambda sec: partial(synth.edge_tape, sec_level=sec)  # noqa: E731
    common.check_prove_parity(L, B=2, N=5, seed=seed, sec_level=sec_prove, make_tape=edge(sec_prove))
    common.check_verify_parity(L, N=5, seed=seed + 1, tampers=6, sec_level=sec_verify, make_tape=edge(sec_verify),
                               make_vtape=VT.edge_verify_tape)
    import test_verify_aggregate as tva
    tva.check_aggregate(L, B=3, N=6, seed=seed + 2, cs=cs, ks=(33,), make_tape=edge(80), make_vtape=VT.edge_verify_tape)


def test_edge_tapes(hostsim):
    check_edge_tapes(hostsim, 201)


def test_edge_tapes_war256(hostsim_war):
    check_edge_tapes(hostsim_war, 211)


def test_noncanonical_p256_coordinates(hostsim):
    """x + p for a point with a small x: p256_mul_batch and keyToInt treat it as (x, y), as the reference does."""
    common.check_noncanonical_p256(hostsim)


def test_multi_chunk_batches_equal_single_chunk():
    """A batch larger than the pipeline chunk is processed in several passes: same bytes."""
    import os
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    g.build_hostsim()
    os.environ.update(ZKA_TOM_W='10', ZKA_P256_HW='8', ZKA_CHUNK='2')
    try:
        small = ZkaLib(g.HOSTSIM)
    finally:
        os.environ.pop('ZKA_CHUNK', None)
    try:
        big = ZkaLib(g.HOSTSIM)
    finally:
        os.environ.pop('ZKA_TOM_W', None)
        os.environ.pop('ZKA_P256_HW', None)
    assert small.config()['chunk'] == 2 and big.config()['chunk'] > 2
    wl = synth.Workload(B=5, N=4, seed=61)
    outs = []
    for L in (small, big):
        P, _ = common.make_params(L, 61, 20)
        tape = synth.random_tape(5, L.prove_tape_len(4, 20), seed=62)
        proofs, plen, status = common.run_prove(L, P, wl, tape, 20)
        assert (status == 0).all()
        vt = VT.random_verify_tape(5, L.verify_tape_len(4, 20), 4, 20, seed=63)
        ok, st = common.run_verify(L, P, wl.msg_hash, wl.ring, proofs, plen, vt)
        assert (ok == 1).all() and (st == 0).all()
        outs.append((proofs.copy(), plen.copy()))
    assert (outs[0][1] == outs[1][1]).all()
    for b in range(5):
        assert outs[0][0][b, :outs[0][1][b]].tobytes() == outs[1][0][b, :outs[1][1][b]].tobytes()
    # the same three chunks dealt to two lanes (lane 1 runs on its own host thread): same bytes again
    small.set_option('lanes', 2)
    assert small.config()['lanes'] == 2
    P, _ = common.make_params(small, 61, 20)
    tape = synth.random_tape(5, small.prove_tape_len(4, 20), seed=62)
    proofs, plen, status = common.run_prove(small, P, wl, tape, 20)
    assert (status == 0).all() and (plen == outs[0][1]).all() and (proofs == outs[0][0]).all()
    vt = VT.random_verify_tape(5, small.verify_tape_len(4, 20), 4, 20, seed=63)
    ok, st = common.run_verify(small, P, wl.msg_hash, wl.ring, proofs, plen, vt)
    assert (ok == 1).all() and (st == 0).all()


def test_ragged_table_windows_bit_exact():
    """Table window widths that do not divide 256 (the defaults, 22 and 20 bits, do not): the last
    window is narrower.  Same proof bytes and verdicts as the oracle with 11- and 9-bit windows."""
    import os
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    g.build_hostsim()
    os.environ.update(ZKA_TOM_W='11', ZKA_P256_HW='9')
    try:
        L = ZkaLib(g.HOSTSIM)
    finally:
        os.environ.pop('ZKA_TOM_W', None)
        os.environ.pop('ZKA_P256_HW', None)
    assert L.config()['tom_w'] == 11 and L.config()['tom_nwin'] == 24
    common.check_prove_parity(L, B=2, N=5, sec_level=20, seed=71)
    common.check_verify_parity(L, N=5, sec_level=20, seed=72, tampers=6)


def test_equal_keys_share_tables_bit_exact(hostsim):
    """Six proofs over a ring of three: several signers repeat, so the per-key tables are shared
    (KeyDedupTask); every proof still equals the oracle's byte for byte."""
    wl = synth.Workload(B=6, N=3, seed=81)
    assert len({bytes(k) for k in wl.pk}) < 6
    common.check_prove_parity(hostsim, B=6, N=3, sec_level=12, seed=81)


def test_large_ring_block_sums_bit_exact(hostsim):
    """Rings above 1024 entries: the Groth-Kohlweiss ring polynomial is summed in blocks of 1024 entries
    by separate threads (prover GkPolyTask/GkPolyReduceTask, verifier VGkSumTask).  N = 2100 pads to
    4096 = 4 blocks; proof bytes and verdicts (incl. tampered proofs) must equal the oracle's."""
    common.check_prove_parity(hostsim, B=1, N=2100, sec_level=20, seed=91)
    common.check_verify_parity(hostsim, N=2100, sec_level=20, seed=92, tampers=4)
