"""Traceable proofs (include/zkattest.h, "Traceable proofs"): the trace block against its restatement in
tests/trace_rule.py, the traced verifier and the opener, on both host-simulator builds and on the GPU."""
import numpy as np
import pytest

from oracle import flat
from oracle import seed_tape as ST
from oracle.curves import tomEdwards256
import trace_rule as TR
from common import make_params, pg
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT

Q = ST.P256_P
SK = 0x1234567890abcdef1234567890abcdef1234567890abcdef1234567890abcdef


@pytest.fixture(params=['hostsim', 'hostsim_war'])
def lib(request):
    L = request.getfixturevalue(request.param)
    pg(L)
    yield L
    flat.set_proof_group(tomEdwards256)


def _be(v):
    return np.frombuffer(int(v).to_bytes(32, 'big'), np.uint8).copy()


class Case:
    """B rows over a ring of N keys at SecLevel S, proved untraced and traced on the same randomness."""

    def __init__(self, L, B=3, N=5, S=16, seed=11, seeded=False, bad_row=None):
        self.L, self.B, self.N, self.S, self.seeded = L, B, N, S, seeded
        self.P, self.po = make_params(L, seed, S)
        self.digest = TR.params_digest(self.po.NistGroup.h.to_bytes(), self.po.ProofGroup.h.to_bytes(), S)
        self.hp = self.po.ProofGroup.h.to_bytes()
        self.wl = synth.Workload(B=B, N=N, seed=seed)
        if bad_row is not None:
            self.wl.which[bad_row] = N + 1          # outside the ring: the untraced call rejects the row
        self.Y = L.trace_pubkey(_be(SK))
        assert self.Y == TR.pubkey(SK)
        self.Lt = L.prove_tape_len(N, S)
        self.tape = synth.random_tape(B, self.Lt + 128, seed=seed + 1)
        self.seeds = np.frombuffer(bytes(range(32)) * B, np.uint8).reshape(B, 32).copy()
        self.seeds[:, 0] = np.arange(B)
        self.T = L.trace_len()
        self.stride = L.proof_max_len(N, S) + self.T

    def prove(self, traced, tape=None):
        L, wl, B = self.L, self.wl, self.B
        proofs = np.zeros((B, self.stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        st = np.zeros(B, np.int32)
        tape = self.tape if tape is None else tape
        if self.seeded:
            f = L.prove_batch_traced_seeded if traced else L.prove_batch_seeded
            args = (self.P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, self.N, self.seeds, proofs, self.stride, plen, st)
        else:
            f = L.prove_batch_traced if traced else L.prove_batch
            args = (self.P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, self.N, tape, tape.shape[1], proofs, self.stride, plen, st)
        f(*args, *((self.Y,) if traced else ()))
        return proofs, plen, st

    def oracle_block(self, proofs, b, tape=None):
        x = int.from_bytes(self.wl.pk[b, 1:33].tobytes(), 'big') % Q
        if self.seeded:
            r, d = TR.seed_draws(self.seeds[b].tobytes())
        else:
            r, d = TR.tape_draws((self.tape if tape is None else tape)[b].tobytes(), self.Lt)
        return TR.prove_block(self.digest, self.hp, self.Y, self.wl.msg_hash[b].tobytes(), proofs[b, :flat.HEAD_LEN].tobytes(), x, r, d)

    def verify(self, proofs, plen, Y=None, msg=None):
        B = proofs.shape[0]
        ok = np.zeros(B, np.uint8)
        st = np.zeros(B, np.int32)
        msg = self.wl.msg_hash[:B] if msg is None else msg
        vts = self.L.verify_tape_len_ex(self.N, self.S, self.S)
        vt = VT.random_verify_tape(B, vts, self.N, self.S, seed=5)
        self.L.verify_batch_traced(self.P, B, msg, self.wl.ring, self.N, proofs, proofs.shape[1], plen, vt, vts, ok, st, self.S,
                                   self.Y if Y is None else Y)
        return ok, st

    def open(self, proofs, plen, sk=SK, ring=None, msg=None):
        B = proofs.shape[0]
        idx = np.zeros(B, np.uint32)
        st = np.zeros(B, np.int32)
        ring = self.wl.ring if ring is None else ring
        msg = self.wl.msg_hash[:B] if msg is None else msg
        self.L.open_batch(self.P, _be(sk), B, msg, ring, ring.shape[0], proofs, proofs.shape[1], plen, idx, st)
        return idx, st


@pytest.mark.parametrize('seeded', [False, True])
def test_prove_bytes(lib, seeded):
    c = Case(lib, seeded=seeded, bad_row=1)
    p0, l0, s0 = c.prove(False)
    p1, l1, s1 = c.prove(True)
    assert list(s0) == list(s1) and s0[1] == 6 and s0[0] == 0 and s0[2] == 0
    for b in range(c.B):
        if s0[b]:
            assert l1[b] == 0 and not p1[b].any()
            continue
        assert l1[b] == l0[b] + c.T
        assert p1[b, :l0[b]].tobytes() == p0[b, :l0[b]].tobytes()
        assert p1[b, l0[b]:l1[b]].tobytes() == c.oracle_block(p1, b), b
        assert p1[b, l1[b]:].tobytes() == p0[b, l1[b]:].tobytes()   # the padding is the untraced call's


def test_trace_draw_out_of_range(lib):
    c = Case(lib, B=2)
    tape = c.tape.copy()
    tape[1, c.Lt + 64:c.Lt + 96] = 0xff            # draw beta >= q
    p, ln, st = c.prove(True, tape)
    assert list(st) == [0, 5] and ln[1] == 0 and not p[1].any()
    assert p[0, ln[0] - c.T:ln[0]].tobytes() == c.oracle_block(p, 0, tape)


def test_zero_nonce(lib):
    """k = 0 makes C1 the identity: war256 has no encoding for it in a fixed slot (status 7), tomEdwards256 encodes (0, 1)."""
    c = Case(lib, B=1)
    tape = c.tape.copy()
    tape[0, c.Lt:c.Lt + 32] = 0
    p, ln, st = c.prove(True, tape)
    if flat.PROOF_GROUP.name == 'war256':
        assert (st[0], ln[0]) == (7, 0) and not p[0].any()
    else:
        assert st[0] == 0 and p[0, ln[0] - c.T:ln[0]].tobytes() == c.oracle_block(p, 0, tape)


def _traced(c):
    p, ln, st = c.prove(True)
    assert not st.any()
    return p, ln


def _with_block(p, ln, b, block):
    q = p.copy()
    q[b, ln[b] - len(block):ln[b]] = np.frombuffer(block, np.uint8)
    return q


def test_verify_fields_and_parse(lib):
    c = Case(lib, B=2)
    p, ln = _traced(c)
    ok, st = c.verify(p, ln)
    assert list(ok) == [1, 1] and not st.any()
    T, WP, WS = c.T, flat.WP, flat.WS
    good = p[0, ln[0] - T:ln[0]].tobytes()
    other = p[1, ln[1] - T:ln[1]].tobytes()
    # each of the eight fields replaced by another valid value: the block parses and fails a relation
    for f in range(8):
        a, z = (f * WP, (f + 1) * WP) if f < 5 else (5 * WP + (f - 5) * WS, 5 * WP + (f - 4) * WS)
        blk = good[:a] + other[a:z] + good[z:]
        assert TR.relations_hold(c.digest, c.hp, c.Y, c.wl.msg_hash[0].tobytes(), p[0].tobytes(), blk, TR.parse_block(blk)) is False
        ok, st = c.verify(_with_block(p, ln, 0, blk)[:1], ln[:1])
        assert (ok[0], st[0]) == (0, 0), f
    # malformed blocks: an off-curve point, a scalar >= q, and for tomEdwards256 a coordinate >= p
    bad = [good[:1] + bytes([good[1] ^ 1]) + good[2:],
           good[:5 * WP] + (b'\x00' * (WS - 32)) + Q.to_bytes(32, 'big') + good[5 * WP + WS:]]
    if flat.PROOF_GROUP.name == 'tomEdwards256':
        g = flat.PROOF_GROUP
        bad.append(good[:WP] + b'\x04' + (g.p + 1).to_bytes(WS, 'big') + good[WP + 1 + WS:])
    for blk in bad:
        with pytest.raises(ValueError):
            TR.parse_block(blk)
        q = _with_block(p, ln, 0, blk)
        q[0, 300] ^= 1                                # a defect in the base part too: the block's code still wins
        ok, st = c.verify(q[:1], ln[:1])
        assert (ok[0], st[0]) == (0, 9)
    # truncated block, trailing bytes, a row shorter than a block
    for n in (ln[0] - 1, ln[0] + 1, c.T - 1):
        ok, st = c.verify(p[:1], np.array([n], np.uint32))
        assert (ok[0], st[0]) == (0, 9), n
    # a wrong opener key
    ok, st = c.verify(p, ln, Y=TR.pubkey(SK + 1))
    assert list(ok) == [0, 0] and not st.any()


def test_verify_base_tampers(lib):
    """A defect in the base part gives the untraced verdict and status."""
    c = Case(lib, B=1)
    p, ln = _traced(c)
    base = p[:, :ln[0] - c.T].copy()
    for off in (1, 140, 400, int(ln[0]) - c.T - 3):
        q, b = p.copy(), base.copy()
        q[0, off] ^= 4
        b[0, off] ^= 4
        bl = np.array([ln[0] - c.T], np.uint32)
        vts = c.L.verify_tape_len_ex(c.N, c.S, c.S)
        ok0, st0 = np.zeros(1, np.uint8), np.zeros(1, np.int32)
        vt = VT.random_verify_tape(1, vts, c.N, c.S, seed=5)
        c.L.verify_batch_ex(c.P, 1, c.wl.msg_hash[:1], c.wl.ring, c.N, b, b.shape[1], bl, vt, vts, ok0, st0, c.S)
        ok1, st1 = c.verify(q, ln)
        assert (ok1[0], st1[0]) == (ok0[0], st0[0]), off


def test_open(lib):
    c = Case(lib, B=3, N=5)
    p, ln = _traced(c)
    idx, st = c.open(p, ln)
    assert list(idx) == list(c.wl.which) and not st.any()
    for b in range(c.B):
        got = TR.open_row(c.digest, c.hp, c.Y, SK, c.wl.msg_hash[b].tobytes(), p[b, :ln[b]].tobytes(), c.wl.ring_ints(), c.N)
        assert got == (int(c.wl.which[b]), 0)
    # duplicates: the smallest index; the signer's key moved out of the ring: 13
    ring = c.wl.ring.copy()
    j = int(c.wl.which[0])
    ring[4] = ring[j]
    ring[0] = ring[j]
    idx, st = c.open(p[:1], ln[:1], ring=ring)
    assert (idx[0], st[0]) == (0, 0)
    ring = c.wl.ring.copy()
    ring[j, 31] ^= 1
    idx, st = c.open(p[:1], ln[:1], ring=ring)
    assert (idx[0], st[0]) == (0xFFFFFFFF, 13)
    # a wrong sk: the block is checked under Y = sk g, whose relations it fails (12); a tampered response: 12
    idx, st = c.open(p[:1], ln[:1], sk=SK + 1)
    assert st[0] == 12
    q = p.copy()
    q[0, ln[0] - 1] ^= 1
    idx, st = c.open(q[:1], ln[:1])
    assert (idx[0], st[0]) == (0xFFFFFFFF, 12)
    q[0, ln[0] - c.T + 1] ^= 0x80
    idx, st = c.open(q[:1], ln[:1])
    assert st[0] in (9, 12)


def test_open_signer_not_which(lib):
    """A `which` that is in the ring but not the signer's key: the proof is invalid, and the block still names the
    signer's own key."""
    c = Case(lib, B=1, N=5)
    j = int(c.wl.which[0])
    c.wl.which[0] = (j + 1) % c.N
    p, ln, st = c.prove(True)
    assert st[0] == 0
    idx, st = c.open(p, ln)
    assert (idx[0], st[0]) == (j, 0)
    ring = c.wl.ring.copy()
    ring[j, 0] ^= 1
    idx, st = c.open(p, ln, ring=ring)
    assert (idx[0], st[0]) == (0xFFFFFFFF, 13)


def test_argument_checks(lib):
    from zkp_ecdsa_b200.capi import ZkaError
    c = Case(lib, B=1)
    wl = c.wl
    out = np.zeros((1, c.stride), np.uint8)
    plen, st = np.zeros(1, np.uint32), np.zeros(1, np.int32)
    with pytest.raises(ZkaError):   # tape stride without the four trace draws
        lib.prove_batch_traced(c.P, 1, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, c.N, c.tape[:, :c.Lt].copy(), c.Lt, out, c.stride,
                               plen, st, c.Y)
    with pytest.raises(ZkaError):   # proof stride without the block
        lib.prove_batch_traced(c.P, 1, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, c.N, c.tape, c.tape.shape[1], out, c.stride - 1,
                               plen, st, c.Y)
    badY = bytes([4]) + bytes(flat.WP - 1)
    with pytest.raises(ZkaError):
        lib.prove_batch_traced(c.P, 1, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, c.N, c.tape, c.tape.shape[1], out, c.stride,
                               plen, st, badY)
    with pytest.raises(ZkaError):
        c.verify(out, plen, Y=badY)
    for sk in (0, Q, Q + 5):
        with pytest.raises(ZkaError):
            lib.trace_pubkey(_be(sk))
        with pytest.raises(ZkaError):
            c.open(out, plen, sk=sk)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _gpu_case(eng, B, N, S, seed=21):
    L = eng.lib
    pg(L)
    c = Case(L, B=B, N=N, S=S, seed=seed)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize('group', ['tomEdwards256', 'war256'])
def test_gpu_traced_batch(request, group):
    import torch
    eng = request.getfixturevalue('gpu_engine' if group == 'tomEdwards256' else 'gpu_engine_war')
    L = eng.lib
    c = _gpu_case(eng, 512, 256, 80)
    p0, l0, s0 = c.prove(False)
    assert not s0.any()
    spots = (0, 137, 511)
    L.set_option('chunk', 128)
    L.set_option('host_chunk', 128)
    try:
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            p, ln, st = c.prove(True)                  # host buffers
            assert not st.any() and (ln == l0 + c.T).all()
            for b in spots:
                assert p[b, :l0[b]].tobytes() == p0[b, :l0[b]].tobytes()
                assert p[b, l0[b]:ln[b]].tobytes() == c.oracle_block(p, b)
            # device buffers
            dev = torch.device('cuda', 0)
            wl = c.wl
            d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in (
                ('msg', wl.msg_hash), ('sig', wl.sig), ('pk', wl.pk), ('which', wl.which.view(np.int32)), ('ring', wl.ring),
                ('tape', c.tape))}
            dp = torch.zeros((c.B, c.stride), dtype=torch.uint8, device=dev)
            dl = torch.zeros(c.B, dtype=torch.int32, device=dev)
            ds = torch.zeros(c.B, dtype=torch.int32, device=dev)
            L.prove_batch_traced(c.P, c.B, d['msg'].data_ptr(), d['sig'].data_ptr(), d['pk'].data_ptr(), d['which'].data_ptr(),
                                 d['ring'].data_ptr(), c.N, d['tape'].data_ptr(), c.tape.shape[1], dp.data_ptr(), c.stride, dl.data_ptr(),
                                 ds.data_ptr(), c.Y)
            torch.cuda.synchronize()
            hp = dp.cpu().numpy()
            assert (dl.cpu().numpy().view(np.uint32) == ln).all() and not ds.cpu().numpy().any()
            assert all(hp[b, :ln[b]].tobytes() == p[b, :ln[b]].tobytes() for b in range(c.B))
            # verify and open on the device rows
            vts = L.verify_tape_len_ex(c.N, c.S, c.S)
            dvt = torch.from_numpy(VT.random_verify_tape(c.B, vts, c.N, c.S, seed=5)).to(dev)
            dok = torch.zeros(c.B, dtype=torch.uint8, device=dev)
            dvs = torch.zeros(c.B, dtype=torch.int32, device=dev)
            L.verify_batch_traced(c.P, c.B, d['msg'].data_ptr(), d['ring'].data_ptr(), c.N, dp.data_ptr(), c.stride, dl.data_ptr(),
                                  dvt.data_ptr(), vts, dok.data_ptr(), dvs.data_ptr(), c.S, c.Y)
            didx = torch.zeros(c.B, dtype=torch.int32, device=dev)
            dos = torch.zeros(c.B, dtype=torch.int32, device=dev)
            L.open_batch(c.P, _be(SK), c.B, d['msg'].data_ptr(), d['ring'].data_ptr(), c.N, dp.data_ptr(), c.stride, dl.data_ptr(),
                         didx.data_ptr(), dos.data_ptr())
            torch.cuda.synchronize()
            assert dok.cpu().numpy().all() and not dvs.cpu().numpy().any()
            assert (didx.cpu().numpy().view(np.uint32) == c.wl.which).all() and not dos.cpu().numpy().any()
            ok, vst = c.verify(p, ln)
            assert ok.all() and not vst.any()
            idx, ost = c.open(p, ln)
            assert (idx == c.wl.which).all() and not ost.any()
        # the self-check: the same rows, every row counted by the check
        L.set_option('self_check', 2)
        r0 = L.stat('self_check_rows')
        p2, l2, s2 = c.prove(True)
        assert (l2 == ln).all() and not s2.any()
        assert all(p2[b, :ln[b]].tobytes() == p[b, :ln[b]].tobytes() for b in range(c.B))
        assert L.stat('self_check_rows') - r0 == c.B
    finally:
        L.set_option('self_check', 1)
        L.set_option('lanes', 3)
        L.set_option('chunk', 4096)
        L.set_option('host_chunk', 2048)
        flat.set_proof_group(tomEdwards256)
    L.params_destroy(c.P)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [2100, 1 << 20])
def test_gpu_open_large_ring(gpu_engine, N):
    L = gpu_engine.lib
    pg(L)
    c = _gpu_case(gpu_engine, 8, 6, 16, seed=31)
    p, ln = _traced(c)
    rng = np.random.default_rng(N)
    ring = rng.integers(0, 256, size=(N, 32), dtype=np.uint8)
    where = [N - 1, 7, N // 2, 0, 5, N - 2, 1, 3]
    for b in range(c.B):
        ring[where[b]] = c.wl.ring[c.wl.which[b]]
    idx, st = c.open(p, ln, ring=ring)
    exp = [int(np.flatnonzero((ring == c.wl.ring[c.wl.which[b]]).all(axis=1))[0]) for b in range(c.B)]
    assert list(idx) == exp and not st.any()
    L.params_destroy(c.P)
