"""Shared g-parts of the prover's commitment walks (GpartLayout, zk_ops.cuh).

A commitment v*g + r*h continues from a g-part v*g computed once per distinct value: C4 of MultProofs 1..3 takes the
g-part of C10, C11, C13 (its value x y is theirs), C4 of MultProof 0 (x y = 1, or 0 when x1 = x2) and every value of 0 or
1 start at their value's window-0 entry, and of the Groth-Kohlweiss commitments only ca_i and cd_i are walked over g
(cl_i commits l_i in {0, 1}, cb_i commits l_i a_i).  The bytes stay the oracle's: batched proofs (one ring and a ring set
mixing depths), the stand-alone pointAdd prover with P = Q (i7 = i8 = 0) and P != Q, and the stand-alone membership
prover with both bit values of `which` in every round.  Host simulators of both proof groups, then the GPU, where the
profile shows how many walks ran.
"""
import numpy as np
import pytest

import common
import test_rings as TR
import test_subproofs as TS
from oracle import commit as OC
from oracle import exp as OE
from oracle import flat
from oracle.big import Tape
from oracle.curves import p256
from zkp_ecdsa_b200 import synth


def check_pointadd(L, same, seed):
    """zka_prove_pointadd_batch on rows with Q = P (same[b]) or Q != P == the oracle's proofPointAdd bytes."""
    tom = common.pg(L)
    P, po = common.make_params(L, seed, 8)
    params = po.ProofGroup
    d = synth.Drbg(seed, 'gpart-pointadd')
    B = len(same)
    tape = synth.random_tape(B, 32 * 38, seed=seed + 1)
    bl = synth.random_tape(B, 32 * 6, seed=seed + 2)
    i32 = lambda v: int(v).to_bytes(32, 'big')   # noqa: E731
    rows, blind, want_pf, want_com = [], [], [], []
    for b in range(B):
        r = [int.from_bytes(bl[b, 32 * i:32 * i + 32].tobytes(), 'big') for i in range(6)]
        Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Qp = Pp if same[b] else p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Rp = Pp.add(Qp)
        cs = [OC.Commitment(params.h.dblmul(tom.new_scalar(rr), params.g, tom.new_scalar(v)), tom.new_scalar(rr))
              for v, rr in zip([c for pt in (Pp, Qp, Rp) for c in pt.to_affine()], r)]
        pi = OE.prove_point_add(params, Pp, Qp, Rp, *cs, Tape(tape[b].tobytes()))
        rows.append(flat._pt(Pp, 65) + flat._pt(Qp, 65) + flat._pt(Rp, 65))
        blind.append(b''.join(i32(v) for v in r))
        want_pf.append(flat.ser_point_add(pi))
        want_com.append(b''.join(c.p.to_bytes() for c in cs))
    arr = lambda rr: np.array([list(x) for x in rr], np.uint8)   # noqa: E731
    com, proofs, st = L.prove_sub_batch('pointadd', P, arr(rows), tape, arr(blind))
    for b in range(B):
        assert st[b] == 0 and proofs[b].tobytes() == want_pf[b] and com[b].tobytes() == want_com[b], (b, same[b])
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------- host simulators
def test_batched_proofs_hostsim(hostsim):
    common.check_prove_parity(hostsim, B=3, N=6, seed=211, sec_level=16)


def test_batched_proofs_hostsim_war(hostsim_war):
    common.check_prove_parity(hostsim_war, B=2, N=5, seed=212, sec_level=16)


def test_ring_set_mixing_depths_hostsim(hostsim):
    TR.check_prove_parity(hostsim, sizes=[2, 5, 17, 40], ring_of=[3, 0, 2, 1, 3, 0], S=16, seed=213)


def test_ring_set_mixing_depths_hostsim_war(hostsim_war):
    TR.check_prove_parity(hostsim_war, sizes=[2, 9, 33], ring_of=[2, 0, 1, 2], S=16, seed=214)


def test_pointadd_doubling_hostsim(hostsim):
    check_pointadd(hostsim, [True, False, True], seed=215)


def test_pointadd_hostsim_war(hostsim_war):
    # P != Q only: with P = Q the war256 build's stand-alone pointAdd proof already differed from the oracle's before the
    # g-parts were shared (from the responses of its first MultProof on), a defect of its own
    check_pointadd(hostsim_war, [False, False], seed=216)


def test_membership_both_bits_hostsim(hostsim):
    # ring of 8: index 0 has l_i = 0 and index 7 l_i = 1 in every round, 5 mixes them
    TS.check_prove_membership(hostsim, [10 ** 20 + 7 * i for i in range(8)], [0, 7, 5], seed=217)


def test_membership_both_bits_hostsim_war(hostsim_war):
    TS.check_prove_membership(hostsim_war, [10 ** 20 + 7 * i for i in range(8)], [7, 0], seed=218)


# ------------------------------------------------------------------------------------------------------ GPU
def _items(prof, name):
    return sum(e['items'] for k, e in prof.items() if k.split('::')[-1] == name)


@pytest.mark.gpu
def test_gpart_reuse_on_gpu(gpu_engine):
    """The oracle's bytes, and the profile counts 24 g-walks per item plus 2 per GK round: the sharing is live."""
    L = gpu_engine.lib
    B, N, S, seed = 6, 40, 80, 219
    P, po = common.make_params(L, seed, S)
    wl = synth.Workload(B=B, N=N, seed=seed)
    tape = synth.random_tape(B, L.prove_tape_len(N, S), seed=seed + 100)
    L.set_profiling(True)
    L.profile_reset()
    try:
        proofs, plen, status = common.run_prove(L, P, wl, tape, S)
        prof = L.profile()
    finally:
        L.set_profiling(False)
    assert (status == 0).all(), status
    n = (N - 1).bit_length()
    M = 0
    for b in range(B):
        pr, _ = common.oracle_proof(po, wl, tape, b)
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), b
        M += sum(1 for e in pr.expProof if e.alpha is None)
    assert _items(prof, 'TomCommitGTask') == 24 * M + 2 * B * n
    assert _items(prof, 'TomCommitHTask') == 34 * M + 4 * B * n
    L.params_destroy(P)
    TR.check_prove_parity(L, sizes=[2, 5, 17, 300], ring_of=[3, 0, 2, 1, 3, 0, 2], S=16, seed=220)
    check_pointadd(L, [True, False, True, True, False], seed=221)
    TS.check_prove_membership(L, [10 ** 20 + 7 * i for i in range(16)], [0, 15, 5, 10], seed=222)


@pytest.mark.gpu
def test_gpart_reuse_on_gpu_war(gpu_engine_war):
    L = gpu_engine_war.lib
    common.check_prove_parity(L, B=3, N=9, seed=223, sec_level=16)
    check_pointadd(L, [False, False], seed=224)
    TS.check_prove_membership(L, [10 ** 20 + 7 * i for i in range(8)], [0, 7, 5], seed=225)
