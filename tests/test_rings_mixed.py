"""Ring-set rows of different ring depths in ONE pass of the batched pipeline (include/zkattest.h, "ring sets").

A chunk is laid out for the largest depth its call uses and every row follows the depth of its own ring, so the order
of depths in ring_of changes neither a row's bytes, verdict and status (those of the one-ring call on its ring) nor the
number of passes.  Host simulators of both proof groups, then the GPU on the interleaved 8192-row set of
tools/rings_mixed_bench.py.
"""
import numpy as np
import pytest

import common
import test_rings as TR
from oracle import flat
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT

SIZES = [2, 5, 8, 17, 300]               # depths 1, 3, 3, 5, 9
RING_OF = [4, 0, 1, 3, 2, 4, 0, 3]       # depths 9 1 3 5 3 9 1 5: another depth on every row
DEPTH = [VT.ceil_log2(s) for s in SIZES]


def _changes_every_row(ring_of, depth=DEPTH):
    d = [depth[int(r)] for r in ring_of]
    return all(a != b for a, b in zip(d, d[1:]))


def _by_depth(ring_of, depth=DEPTH):
    return np.array(sorted(range(len(ring_of)), key=lambda b: (depth[int(ring_of[b])], b)))


# ---------------------------------------------------------------------------------------------------- 1. bytes
def check_bytes(L, ring_of, S, seed):
    assert _changes_every_row(ring_of)
    # the oracle on every row (3 + 4S + 40Z + 5 n_r draws, proof_len) and the same rows in a shuffled order
    wl, proofs, plen = TR.check_prove_parity(L, sizes=SIZES, ring_of=ring_of, S=S, seed=seed)
    P, _ = common.make_params(L, seed, S)
    rs = TR.Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(SIZES), S), seed=seed + 100)     # check_prove_parity's tape
    # each row equals the one-ring call on its ring
    for r in sorted(set(int(x) for x in ring_of)):
        rows = np.flatnonzero(wl.ring_of == r)
        rp, rl, rst = common.run_prove(L, P, TR._one_ring(wl, rows, r), tape[rows][:, :L.prove_tape_len(SIZES[r], S)].copy(), S)
        assert (rst == 0).all()
        for i, b in enumerate(rows):
            assert proofs[b, :plen[b]].tobytes() == rp[i, :rl[i]].tobytes(), (r, b)
    # the rows sorted by depth give the same bytes per row
    order = _by_depth(wl.ring_of)
    p2, l2, s2 = TR.prove_rings(L, P, rs, TR._rows(wl, order), tape[order].copy(), S)
    assert (s2 == 0).all()
    for i, b in enumerate(order):
        assert p2[i, :l2[i]].tobytes() == proofs[b, :plen[b]].tobytes(), (i, b)
    # seeded: each row's proof is the tape proof on zka_seed_tape's expansion for its own ring size
    seeds = TR._seeds(wl.B, f'mixed{seed}')
    sp, sl, sst = TR.prove_rings_seeded(L, P, rs, wl, seeds, S)
    stape = TR.row_seed_tape(L, 0, seeds, SIZES, wl.ring_of, S)
    tp, tl, ts = TR.prove_rings(L, P, rs, wl, stape, S)
    assert (sst == 0).all() and (ts == 0).all() and np.array_equal(sl, tl)
    for b in range(wl.B):
        assert sp[b, :sl[b]].tobytes() == tp[b, :tl[b]].tobytes(), b
    rs.close()
    L.params_destroy(P)


def test_mixed_bytes_hostsim_s16(hostsim):
    check_bytes(hostsim, RING_OF, 16, 131)


def test_mixed_bytes_hostsim_s80(hostsim):
    check_bytes(hostsim, [4, 0, 3], 80, 132)


def test_mixed_bytes_hostsim_war(hostsim_war):
    check_bytes(hostsim_war, [3, 4, 0, 1, 4], 16, 133)


# ------------------------------------------------------------------------------------------------- 2. one pass
def test_mixed_call_is_one_pass_hostsim(hostsim):
    """64 rows whose depth alternates launch exactly what the same rows grouped by depth launch, and what ONE one-ring call
    over 64 rows launches (the chunk holds them all): no pass per run of equal depth."""
    L, S, K, seed = hostsim, 2, 2, 134
    sizes = [2, 17]
    ring_of = np.arange(64) % 2
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(64, sizes, ring_of, seed=seed)
    rs = TR.Set(L, wl)
    tape = synth.random_tape(64, L.prove_tape_len(17, S), seed=seed)
    vt = TR.row_verify_tape(sizes, ring_of, S, K, seed)

    def launches(fn):
        n = L.launch_count()
        out = fn()
        return L.launch_count() - n, out
    n_il, (proofs, plen, st) = launches(lambda: TR.prove_rings(L, P, rs, wl, tape, S))
    assert (st == 0).all()
    order = _by_depth(ring_of, [1, 5])
    n_gr, _ = launches(lambda: TR.prove_rings(L, P, rs, TR._rows(wl, order), tape[order].copy(), S))
    one = TR._one_ring(wl, np.flatnonzero(ring_of == 1), 1)
    n_one, _ = launches(lambda: common.run_prove(L, P, one, tape[ring_of == 1].copy(), S))
    assert n_il == n_gr
    assert n_il <= n_one + 2          # a one-ring call also prepares its ring and its Lagrange matrix
    v_il, (ok, vst) = launches(lambda: TR.verify_rings(L, P, rs, ring_of, wl.msg_hash, proofs, plen, vt, K))
    assert ok.all() and not vst.any()
    v_gr, (ok, vst) = launches(lambda: TR.verify_rings(L, P, rs, ring_of[order], wl.msg_hash[order], proofs[order], plen[order],
                                                       vt[order], K))
    assert ok.all() and not vst.any() and v_il == v_gr
    rs.close()
    L.params_destroy(P)


# -------------------------------------------------------------------------------------------------- 3. verdicts
def _patched(monkeypatch):
    monkeypatch.setattr(TR, 'SIZES', SIZES)
    monkeypatch.setattr(TR, 'RING_OF', RING_OF)


def test_mixed_verify_matches_oracle_hostsim(hostsim, monkeypatch):
    """test_rings' tamper set on the interleaved batch: flipped bits, truncations, wrong messages, and a proof for the ring of
    8 verified against the rings of 17, 2 and 300 (other depths: the GK length check fails, verdict false)."""
    _patched(monkeypatch)
    TR.check_verify_parity(hostsim, seed=135)


def test_mixed_verify_matches_oracle_hostsim_war(hostsim_war, monkeypatch):
    _patched(monkeypatch)
    TR.check_verify_parity(hostsim_war, seed=136, tampers=4)


def test_mixed_gk_draw_out_of_range_on_a_shallow_row(hostsim):
    """A GK drain >= the group order in a depth-1 row between rows of depth 9 and 5: that row gets the status of the
    one-ring call on its ring, its neighbours are accepted; the same draw index is an exp drain or index byte for nobody."""
    L, S, K, seed = hostsim, 16, 5, 137
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(RING_OF), SIZES, RING_OF, seed=seed)
    rs = TR.Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(SIZES), S), seed=seed)
    proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
    assert (st == 0).all()
    vt = TR.row_verify_tape(SIZES, wl.ring_of, S, K, seed)
    b = 1
    assert wl.ring_of[b] == 0 and DEPTH[0] == 1
    vt[b, 64:96] = 0xff                                     # relFinal, the last of the row's 2 n_r + 1 = 3 GK drains
    ok, vst = TR.verify_rings(L, P, rs, wl.ring_of, wl.msg_hash, proofs, plen, vt, K)
    ok1, st1 = np.zeros(1, np.uint8), np.zeros(1, np.int32)
    vts = L.verify_tape_len_ex(SIZES[0], S, K)
    L.verify_batch_ex(P, 1, wl.msg_hash[b:b + 1].copy(), wl.rings[0], SIZES[0], proofs[b:b + 1].copy(), proofs.shape[1],
                      plen[b:b + 1].copy(), vt[b:b + 1, :vts].copy(), vts, ok1, st1, K)
    assert st1[0] != 0 and vst[b] == st1[0] and ok[b] == ok1[0] == 0
    assert list(np.delete(ok, b)) == [1] * (wl.B - 1) and not np.delete(vst, b).any()
    rs.close()
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------------- 4. aggregate
def test_mixed_chunk_on_the_aggregate_path_hostsim(hostsim):
    L, S, K, seed = hostsim, 16, 5, 138
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(RING_OF), SIZES, RING_OF, seed=seed)
    rs = TR.Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(SIZES), S), seed=seed)
    proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
    assert (st == 0).all()
    vt = TR.row_verify_tape(SIZES, wl.ring_of, S, K, seed)
    B = wl.B
    verify = lambda pr, ln: TR.verify_rings(L, P, rs, wl.ring_of, wl.msg_hash, pr, ln, vt, K)   # noqa: E731
    try:
        for c in (0, 4):
            if c:
                L.set_option('agg_c', c)
            p0, f0 = L.stat('agg_pass'), L.stat('agg_fail')
            ok, vst = verify(proofs, plen)
            assert ok.all() and not vst.any(), (c, ok, vst)
            assert L.stat('agg_pass') > p0 and L.stat('agg_fail') == f0, c
            # one wrong row (its last GK response, in the shallow row between two deep ones): per-proof verdicts
            bad = proofs.copy()
            bad[1, plen[1] - 1] ^= 1
            ok, vst = verify(bad, plen)
            assert L.stat('agg_fail') > f0
            L.set_option('agg', 1)
            ok2, vst2 = verify(bad, plen)
            L.set_option('agg', 2)
            assert np.array_equal(ok, ok2) and np.array_equal(vst, vst2)
            assert ok[1] == 0 and list(np.delete(ok, 1)) == [1] * (B - 1) and not vst.any()
            # one malformed row: its own status, the others accepted
            short = plen.copy()
            short[4] -= 3
            ok, vst = verify(proofs, short)
            assert ok[4] == 0 and vst[4] != 0 and list(np.delete(ok, 4)) == [1] * (B - 1) and not np.delete(vst, 4).any()
    finally:
        L.set_option('agg', 2)
        L.set_option('agg_c', 6)
        rs.close()
        L.params_destroy(P)


# ----------------------------------------------------------------------------------- 6. host buffers, short strides
def test_mixed_strides_cover_the_largest_ring_used(hostsim):
    L, S, seed = hostsim, 16, 139
    P, _ = common.make_params(L, seed, S)
    ring_of = np.array([3, 0, 1, 3, 0], np.uint32)          # the ring of 300 is in the set and not used
    wl = synth.RingsWorkload(len(ring_of), SIZES, ring_of, seed=seed)
    rs = TR.Set(L, wl)
    ts, ps = L.prove_tape_len(17, S), L.proof_max_len(17, S)
    tape = synth.random_tape(wl.B, ts, seed=seed)

    def prove(tape_stride, proof_stride):
        proofs, plen, st = np.zeros((wl.B, ps), np.uint8), np.zeros(wl.B, np.uint32), np.zeros(wl.B, np.int32)
        L.prove_batch_rings(P, rs.h, wl.ring_of, wl.B, wl.msg_hash, wl.sig, wl.pk, wl.which, tape, tape_stride, proofs, proof_stride,
                            plen, st)
        return proofs, plen, st
    proofs, plen, st = prove(ts, ps)
    assert (st == 0).all() and plen.all()
    with pytest.raises(Exception):
        prove(ts, ps - 1)
    with pytest.raises(Exception):
        prove(32 * (3 + 4 * S + 5 * 5) - 1, ps)              # the draws before any item at the largest depth used, less a byte
    K = 5
    vt = TR.row_verify_tape(SIZES, ring_of, S, K, seed)
    assert vt.shape[1] == L.verify_tape_len_ex(17, S, K)
    ok, vst = TR.verify_rings(L, P, rs, ring_of, wl.msg_hash, proofs, plen, vt, K)
    assert ok.all() and not vst.any()
    okb, stb = np.zeros(wl.B, np.uint8), np.zeros(wl.B, np.int32)
    with pytest.raises(Exception):
        L.verify_batch_rings(P, rs.h, wl.ring_of, wl.B, wl.msg_hash, proofs, ps, plen, vt, vt.shape[1] - 1, K, okb, stb)
    rs.close()
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------------ 7. progress flags
def test_mixed_call_writes_progress_flags(hostsim):
    """A ring-set call has the chunk schedule of the one-ring call over the same B: one flag per chunk, all set at return."""
    L, S, seed = hostsim, 2, 140
    P, _ = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(len(RING_OF), SIZES, RING_OF, seed=seed)
    rs = TR.Set(L, wl)
    tape = synth.random_tape(wl.B, L.prove_tape_len(max(SIZES), S), seed=seed)
    cfg = L.config()
    flags = np.zeros(16, np.uint32)
    try:
        L.set_option('chunk', 3)
        L.set_option('host_chunk', 3)
        off = L.chunk_schedule(wl.B, host_buffers=True)
        assert off[0] == 0 and off[-1] == wl.B and len(off) - 1 >= 3
        L.set_progress(flags)
        proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
        assert (st == 0).all()
        assert list(flags) == [1] * (len(off) - 1) + [0] * (flags.size - len(off) + 1)
    finally:
        L.set_progress(None)
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)
    whole, wlen, _ = TR.prove_rings(L, P, rs, wl, tape, S)
    assert np.array_equal(plen, wlen)                                        # chunks of 3 rows: the same bytes
    assert all(proofs[b, :plen[b]].tobytes() == whole[b, :plen[b]].tobytes() for b in range(wl.B))
    rs.close()
    L.params_destroy(P)


# ------------------------------------------------------------------------------------------------------------- GPU
def mixed_gpu_set(B=8192):
    """The 64 rings of 8 .. 1024 of tools/rings_bench.py case b, a ring of 2100 (depth 12: the blocked GK kernels) and a ring
    of 2; ring_of walks the rings so that the depth changes on every row."""
    sizes = [8 << (i % 8) for i in range(64)] + [2100, 2]
    depth = [VT.ceil_log2(s) for s in sizes]
    ring_of = np.arange(B, dtype=np.uint32) % 66
    assert _changes_every_row(ring_of, depth)
    return sizes, depth, ring_of


def _dev_prove(L, P, rs, wl, tape, ps):
    import torch
    B = wl.B
    dp = torch.zeros(B * ps, dtype=torch.uint8, device='cuda')
    dl = torch.zeros(B, dtype=torch.int32, device='cuda')
    ds = torch.zeros(B, dtype=torch.int32, device='cuda')
    dro, dm, dsig, dpk, dw, dt = (TR._dev(x) for x in (wl.ring_of.view(np.int32), wl.msg_hash, wl.sig, wl.pk, wl.which.view(np.int32), tape))
    L.prove_batch_rings(P, rs.h, dro.data_ptr(), B, dm.data_ptr(), dsig.data_ptr(), dpk.data_ptr(), dw.data_ptr(), dt.data_ptr(),
                        tape.shape[1], dp.data_ptr(), ps, dl.data_ptr(), ds.data_ptr())
    torch.cuda.synchronize()
    return dp.cpu().numpy().reshape(B, ps), dl.cpu().numpy().view(np.uint32), ds.cpu().numpy()


def check_gpu_mixed(L, B, S, seed, K=20):
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    sizes, depth, ring_of = mixed_gpu_set(B)
    P, po = common.make_params(L, seed, S)
    wl = synth.RingsWorkload(B, sizes, ring_of, seed=seed)
    rs = TR.Set(L, wl)
    Nmax = max(sizes)
    tape = synth.random_tape(B, L.prove_tape_len(Nmax, S), seed=seed + 1)
    ps = L.proof_max_len(Nmax, S)
    order = _by_depth(ring_of, depth)
    srt = TR._rows(wl, order)
    cfg = L.config()
    ref = rlen = None
    try:
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            for chunk in (None, 128):
                if chunk:
                    L.set_option('chunk', chunk)
                    L.set_option('host_chunk', chunk)
                if ref is None:
                    # the depth-sorted call: the reference of every other run; the profile counts one GkPolyTask per chunk
                    L.set_profiling(True)
                    L.profile_reset()
                    sp, sl, sst = TR.prove_rings(L, P, rs, srt, tape[order].copy(), S)
                    assert (sst == 0).all()
                    ref, rlen = np.zeros_like(sp), np.zeros_like(sl)
                    ref[order], rlen[order] = sp, sl
                    del sp
                    L.profile_reset()
                    proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
                    prof = L.profile()
                    L.set_profiling(False)
                    gk = [v for k, v in prof.items() if k.endswith('GkPolyTask')]
                    assert len(gk) == 1 and gk[0]['launches'] == len(L.chunk_schedule(B, host_buffers=True)) - 1, prof.keys()
                else:
                    proofs, plen, st = TR.prove_rings(L, P, rs, wl, tape, S)
                assert (st == 0).all() and np.array_equal(plen, rlen), ('host', lanes, chunk)
                assert all(proofs[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes() for b in range(B)), ('host', lanes, chunk)
                got, gl, gs = _dev_prove(L, P, rs, wl, tape, ps)
                assert not gs.any() and np.array_equal(gl, rlen), ('device', lanes, chunk)
                assert all(got[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes() for b in range(B)), ('device', lanes, chunk)
                del proofs, got
                L.set_option('chunk', cfg['chunk'])
                L.set_option('host_chunk', 2048)
        # verification: every row accepted (aggregate path), then one tampered row per chunk of 128 is the only rejection
        vt = TR.row_verify_tape(sizes, ring_of, S, K, seed)
        tampered = np.arange(5, B, 128)
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            passed = L.stat('agg_pass')
            ok, vst = TR.verify_rings(L, P, rs, ring_of, wl.msg_hash, ref, rlen, vt, K)
            assert ok.all() and not vst.any()
            assert L.stat('agg_pass') > passed
            L.set_option('chunk', 128)
            L.set_option('host_chunk', 128)
            ref[tampered, 300] ^= 1
            ok, vst = TR.verify_rings(L, P, rs, ring_of, wl.msg_hash, ref, rlen, vt, K)
            ref[tampered, 300] ^= 1
            L.set_option('chunk', cfg['chunk'])
            L.set_option('host_chunk', 2048)
            assert not ok[tampered].any() and ok.sum() == B - len(tampered) and not np.delete(vst, tampered).any()
    finally:
        L.set_profiling(False)
        L.set_option('lanes', cfg['lanes'])
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)
    spots = [0, 7, 64, 65]                                   # rings of 8, 1024, 2100 and 2
    if L.group != 'tomEdwards256':     # oracle/cpu restates the tomEdwards256 build: the Python oracle checks war256
        for b in spots:
            pr, _ = TR.oracle_row(po, wl, b, tape[b].tobytes())
            assert ref[b, :rlen[b]].tobytes() == flat.ser_proof(pr), b
    else:
        g.build_oracle_cpu()
        cpu = ZkaLib(g.ORACLE_CPU)
        hn, hp = cpu.params_generate(synth.params_rnd(seed))
        Pc = cpu.params_create(hn, hp, S)
        for b in spots:
            r = int(ring_of[b])
            cp, cl, cs = common.run_prove(cpu, Pc, TR._one_ring(wl, [b], r), tape[[b]][:, :L.prove_tape_len(sizes[r], S)].copy(), S)
            assert cs[0] == 0 and cp[0, :cl[0]].tobytes() == ref[b, :rlen[b]].tobytes(), b
        cpu.params_destroy(Pc)
    rs.close()
    L.params_destroy(P)


@pytest.mark.gpu
def test_mixed_depths_on_gpu(gpu_engine):
    check_gpu_mixed(gpu_engine.lib, 8192, S=80, seed=141)


@pytest.mark.gpu
def test_mixed_depths_on_gpu_war(gpu_engine_war):
    check_gpu_mixed(gpu_engine_war.lib, 8192, S=20, seed=142)
