"""Seeded randomness: the tape a 32-byte seed stands for (include/zkattest.h, "Seeded randomness"), expanded on the device.

The expansion is checked against its restatement in oracle/seed_tape.py (itself checked against RFC 8439 and the
`cryptography` package), and a seeded call against the tape call on the expanded tape and against the oracle, on the
host simulator (both proof groups) and on the GPU.
"""
import ctypes as C
import os
import struct

import numpy as np
import pytest

import common
from oracle import flat
from oracle import seed_tape as ST
from oracle import zkattest as OZ
from oracle.big import Tape
from zkp_ecdsa_b200 import api, synth
from zkp_ecdsa_b200 import verify_tape as VT


def _seeds(rows, tag):
    return np.frombuffer(synth.Drbg(rows, f'seeds-{tag}').bytes(32 * rows), np.uint8).reshape(rows, 32).copy()


def _n(N):
    return VT.ceil_log2(N)


# ------------------------------------------------------------------------------------------------- the PRF itself
def test_chacha20_rfc8439_block_vector():
    # RFC 8439 2.3.2
    key = bytes(range(32))
    nonce = bytes.fromhex('000000090000004a00000000')
    want = bytes.fromhex('10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e'
                         'd2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e')
    assert ST.chacha20_block(key, 1, nonce) == want


def test_chacha20_matches_cryptography():
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    d = synth.Drbg(0, 'chacha')
    for i in range(24):
        key, nonce = d.bytes(32), d.bytes(12)
        ctr = int.from_bytes(d.bytes(4), 'little') if i % 3 else i
        ctr = min(ctr, 0xffffffff - 2)
        enc = Cipher(algorithms.ChaCha20(key, struct.pack('<I', ctr) + nonce), mode=None).encryptor()
        ks = enc.update(bytes(192))
        for j in range(3):
            assert ST.chacha20_block(key, ctr + j, nonce) == ks[64 * j:64 * j + 64], (i, j)


# ------------------------------------------------------------------------------------------- zka_seed_tape vs oracle
def check_seed_tapes(L, cases):
    for S, N, Ks in cases:
        seeds = _seeds(2, f'{S}-{N}')
        n = _n(N)
        pt = L.seed_tape(0, seeds, N, S)
        assert pt.shape[1] == L.prove_tape_len(N, S)
        for b in range(2):
            assert pt[b].tobytes() == ST.prove_tape(seeds[b].tobytes(), S, n), ('prove', S, N, b)
        for K in Ks:
            vt = L.seed_tape(1, seeds, N, S, K)
            assert vt.shape[1] == L.verify_tape_len_ex(N, S, K)
            for b in range(2):
                assert vt[b].tobytes() == ST.verify_tape(seeds[b].tobytes(), n, S, K), ('verify', S, N, K, b)
        assert not np.array_equal(pt[0], pt[1])


SEED_TAPE_CASES = [(16, N, (5,)) for N in (2, 6, 17, 256)] + [(80, N, (5, 20, 80)) for N in (2, 6, 17, 256)]


def test_seed_tape_matches_oracle_hostsim(hostsim):
    check_seed_tapes(hostsim, SEED_TAPE_CASES)


def test_seed_tape_matches_oracle_hostsim_war(hostsim_war):
    check_seed_tapes(hostsim_war, [(16, 6, (5,)), (80, 17, (20,))])


# --------------------------------------------------------------------- the 32-byte draw with a caller-given modulus
class SeedProbe:
    def __init__(self, path):
        self.lib = C.CDLL(path)
        self.lib.probe_seed_draw.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]

    def draw(self, seeds, domain, index, mod):
        m = np.array([(mod >> (32 * j)) & 0xffffffff for j in range(8)], np.uint32)
        idx = np.asarray(index, np.uint64)
        out = np.zeros((len(seeds), 32), np.uint8)
        assert self.lib.probe_seed_draw(len(seeds), seeds.ctypes.data, domain, idx.ctypes.data, m.ctypes.data,
                                        out.ctypes.data) == 0
        return out


REJECTION_MODULI = [(1 << 255) + 1, 3 << 254, ST.P256_N, ST.P256_P]


def check_probe(pr):
    seeds = _seeds(64, 'probe')
    index = [(i * 0x9e3779b97f4a7c15) & ((1 << 64) - 1) for i in range(64)]
    rejected = 0
    for mod in REJECTION_MODULI:
        for dom in (1, 2):
            out = pr.draw(seeds, dom, index, mod)
            for i in range(64):
                src = ST.Stream(seeds[i].tobytes(), dom, index[i])
                want = ST.rnd(src, mod).to_bytes(32, 'big')
                assert out[i].tobytes() == want, (hex(mod), dom, i)
                first = ST.Stream(seeds[i].tobytes(), dom, index[i]).fill(32)
                rejected += first != want
    assert rejected > 40     # the rejection branch ran (about half the candidates fail for the first two moduli)
    lo = np.zeros(8, np.uint32)
    lo[7] = 0x7fffffff      # moduli below 2^255 are refused
    assert pr.lib.probe_seed_draw(1, seeds.ctypes.data, 1, np.zeros(1, np.uint64).ctypes.data, lo.ctypes.data,
                                  np.zeros(32, np.uint8).ctypes.data) == -1


def test_draw_rejection_branch_host():
    import __graft_entry__ as g
    g.build_probe_seed(host=True)
    check_probe(SeedProbe(g.PROBE_SEED_HOST))


@pytest.mark.gpu
def test_draw_rejection_branch_device():
    import __graft_entry__ as g
    g.build_probe_seed()
    check_probe(SeedProbe(g.PROBE_SEED))


# --------------------------------------------------------------------------------------------- seeded prove / verify
def run_prove_seeded(L, P, wl, seeds, sec_level):
    B, N = wl.B, wl.N
    ps = L.proof_max_len(N, sec_level)
    proofs = np.zeros((B, ps), np.uint8)
    plen = np.zeros(B, np.uint32)
    status = np.zeros(B, np.int32)
    L.prove_batch_seeded(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, seeds, proofs, ps, plen, status)
    return proofs, plen, status


def check_seeded_prove(L, B, N, sec_level, seed):
    P, po = common.make_params(L, seed, sec_level)
    wl = synth.Workload(B=B, N=N, seed=seed)
    seeds = _seeds(B, f'prove-{seed}')
    proofs, plen, status = run_prove_seeded(L, P, wl, seeds, sec_level)
    assert (status == 0).all(), status
    tape = L.seed_tape(0, seeds, N, sec_level)
    tproofs, tplen, tstatus = common.run_prove(L, P, wl, tape, sec_level)
    assert (tstatus == 0).all() and (tplen == plen).all()
    n = _n(N)
    for b in range(B):
        assert proofs[b, :plen[b]].tobytes() == tproofs[b, :plen[b]].tobytes(), b
        tp = Tape(ST.prove_tape(seeds[b].tobytes(), sec_level, n))
        pr = OZ.prove_signature_list(po, wl.msg_hash[b].tobytes(), wl.sig[b].tobytes(), wl.pk[b].tobytes(),
                                     int(wl.which[b]), wl.ring_ints(), tp)
        assert proofs[b, :plen[b]].tobytes() == flat.ser_proof(pr), f'proof {b} differs from the oracle'
        z = sum(1 for e in pr.expProof if e.alpha is None)
        assert tp.calls == 3 + 4 * sec_level + 40 * z + 5 * n
    # the same seeds give the same bytes; other seeds other proofs
    again, plen2, _ = run_prove_seeded(L, P, wl, seeds, sec_level)
    assert (plen2 == plen).all() and np.array_equal(again, proofs)
    other, plen3, st3 = run_prove_seeded(L, P, wl, _seeds(B, f'other-{seed}'), sec_level)
    assert (st3 == 0).all() and all(other[b, :plen3[b]].tobytes() != proofs[b, :plen[b]].tobytes() for b in range(B))
    L.params_destroy(P)


def test_seeded_prove_hostsim_ring6_s80(hostsim):
    check_seeded_prove(hostsim, B=1, N=6, sec_level=80, seed=61)


def test_seeded_prove_hostsim_ring17_s16(hostsim):
    check_seeded_prove(hostsim, B=2, N=17, sec_level=16, seed=62)


def test_seeded_prove_hostsim_war(hostsim_war):
    check_seeded_prove(hostsim_war, B=2, N=6, sec_level=16, seed=63)
    check_seeded_prove(hostsim_war, B=1, N=17, sec_level=80, seed=64)


def tamper_cases(L, wl, good, N, seed, tampers):
    """(proof, msg, ring) cases in the style of common.check_verify_parity"""
    rng = np.random.default_rng(seed)
    ln = len(good)
    cases = []
    for k in range(tampers):
        p, msg, ring = good.copy(), wl.msg_hash[0].copy(), wl.ring.copy()
        kind = k % 8
        if kind < 3:
            p[int(rng.integers(0, ln))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 3:
            p = p[:ln - 1 - int(rng.integers(0, 40))]
        elif kind == 4:
            p[ln - 1 - getattr(L, 'ws', 33) * int(rng.integers(0, 5))] ^= 1
        elif kind == 5:
            msg[int(rng.integers(0, 32))] ^= 1
        elif kind == 6:
            ring[int(wl.which[0]), 31] ^= 1
        else:
            p[int(rng.integers(264, ln - 1200))] ^= 1
        cases.append((p, msg, ring))
    return cases


def check_seeded_verify(L, N=6, sec_level=80, seed=71, tampers=24, K=20):
    P, po = common.make_params(L, seed, sec_level)
    wl = synth.Workload(B=2, N=N, seed=seed)
    proofs, plen, status = run_prove_seeded(L, P, wl, _seeds(2, f'vp-{seed}'), sec_level)
    assert (status == 0).all()
    vs = _seeds(2, f'v-{seed}')
    ok = np.zeros(2, np.uint8)
    st = np.zeros(2, np.int32)
    L.verify_batch_seeded(P, 2, wl.msg_hash, wl.ring, N, proofs, proofs.shape[1], plen, vs, K, ok, st)
    assert list(ok) == [1, 1] and list(st) == [0, 0]
    good = proofs[0, :plen[0]].copy()
    cases = tamper_cases(L, wl, good, N, seed, tampers)
    vseeds = _seeds(len(cases), f'vt-{seed}')
    vtapes = L.seed_tape(1, vseeds, N, sec_level, K)
    n_ok = n_false = n_err = 0
    for k, (p, msg, ring) in enumerate(cases):
        arr = np.zeros((1, max(len(p), 1)), np.uint8)
        arr[0, :len(p)] = p
        pl = np.array([len(p)], np.uint32)
        m = msg.reshape(1, 32).copy()
        ok1, st1 = np.zeros(1, np.uint8), np.zeros(1, np.int32)
        L.verify_batch_seeded(P, 1, m, ring, N, arr, arr.shape[1], pl, vseeds[k:k + 1].copy(), K, ok1, st1)
        ok2, st2 = np.zeros(1, np.uint8), np.zeros(1, np.int32)
        L.verify_batch_ex(P, 1, m, ring, N, arr, arr.shape[1], pl, vtapes[k:k + 1].copy(), vtapes.shape[1], ok2, st2, K)
        assert (ok1[0], st1[0]) == (ok2[0], st2[0]), k
        got = 'err' if st1[0] else bool(ok1[0])
        try:
            prf = flat.de_proof(p.tobytes(), sec_level)
            exp = OZ.verify_signature_list(po, msg.tobytes(), [int.from_bytes(ring[i].tobytes(), 'big') for i in range(N)], prf,
                                           Tape(VT.oracle_stream(vtapes[k].tobytes(), N, sec_level)), K)
        except ValueError:
            exp = 'err'
        assert got == exp, (k, got, int(st1[0]), exp)
        n_ok += exp is True
        n_false += exp is False
        n_err += exp == 'err'
    assert n_false and n_err
    L.params_destroy(P)


def test_seeded_verify_hostsim(hostsim):
    check_seeded_verify(hostsim)


def test_seeded_verify_hostsim_war(hostsim_war):
    check_seeded_verify(hostsim_war, N=5, sec_level=20, seed=72, tampers=8, K=5)


def test_argument_checks_match_the_tape_api(hostsim):
    L = hostsim
    P, _ = common.make_params(L, 73, 16)
    wl = synth.Workload(B=2, N=6, seed=73)
    ps = L.proof_max_len(6, 16)
    proofs, plen, st = np.zeros((2, ps), np.uint8), np.zeros(2, np.uint32), np.zeros(2, np.int32)
    ok = np.zeros(2, np.uint8)
    seeds = _seeds(2, 'args')
    tape = L.seed_tape(0, seeds, 6, 16)
    vt = L.seed_tape(1, seeds, 6, 16, 5)
    p = C.c_void_p
    ptr = lambda a: p(a.ctypes.data)   # noqa: E731
    lib, ctx = L.lib, L.ctx

    def prove(fn, rnd, B=2, N=6):
        if fn == 'seeded':
            return lib.zka_prove_batch_seeded(ctx, P, B, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), N,
                                              rnd, ptr(proofs), ps, ptr(plen), ptr(st))
        return lib.zka_prove_batch(ctx, P, B, ptr(wl.msg_hash), ptr(wl.sig), ptr(wl.pk), ptr(wl.which), ptr(wl.ring), N, rnd,
                                   tape.shape[1], ptr(proofs), ps, ptr(plen), ptr(st))

    def verify(fn, rnd, B=2, N=6):
        if fn == 'seeded':
            return lib.zka_verify_batch_seeded(ctx, P, B, ptr(wl.msg_hash), ptr(wl.ring), N, ptr(proofs), ps, ptr(plen), rnd, 5,
                                               ptr(ok), ptr(st))
        return lib.zka_verify_batch_ex(ctx, P, B, ptr(wl.msg_hash), ptr(wl.ring), N, ptr(proofs), ps, ptr(plen), rnd, vt.shape[1],
                                       ptr(ok), ptr(st), 5)

    for B, N in ((0, 6), (2, 1), (2, (1 << 20) + 1), (2, 6)):
        assert prove('seeded', ptr(seeds), B, N) == prove('tape', ptr(tape), B, N), (B, N)
        assert verify('seeded', ptr(seeds), B, N) == verify('tape', ptr(vt), B, N), (B, N)
    for B in (0, 2):
        assert prove('seeded', p(0), B) == prove('tape', p(0), B) == -1
        assert verify('seeded', p(0), B) == verify('tape', p(0), B) == -1
    out = np.zeros((2, tape.shape[1]), np.uint8)
    assert lib.zka_seed_tape(ctx, 0, 2, p(0), 6, 16, 0, ptr(out), out.shape[1]) == -1
    assert lib.zka_seed_tape(ctx, 2, 2, ptr(seeds), 6, 16, 0, ptr(out), out.shape[1]) == -1
    assert lib.zka_seed_tape(ctx, 0, 2, ptr(seeds), 1, 16, 0, ptr(out), out.shape[1]) == -1
    assert lib.zka_seed_tape(ctx, 0, 2, ptr(seeds), 6, 16, 0, ptr(out), out.shape[1] - 1) == -1
    assert lib.zka_seed_tape(ctx, 1, 2, ptr(seeds), 6, 16, 17, ptr(out), out.shape[1]) == -1   # samples > sec_level
    assert lib.zka_seed_tape(ctx, 0, 0, ptr(seeds), 6, 16, 0, ptr(out), out.shape[1]) == 0
    L.params_destroy(P)


class _Params:
    def __init__(self, handle, sec_level):
        self.handle, self.sec_level = handle, sec_level


def test_engine_default_seeds_come_from_os_urandom(hostsim, monkeypatch):
    """api.Engine's seeded entry points draw os.urandom(32 * B) and touch no numpy generator."""
    eng = api.Engine.__new__(api.Engine)
    eng.lib, eng.proof_group = hostsim, hostsim.group
    P, po = common.make_params(hostsim, 74, 16)
    wl = synth.Workload(B=2, N=5, seed=74)
    drawn = []
    real = os.urandom

    def urandom(n):
        b = real(n)
        drawn.append(b)
        return b

    def no_numpy(*a, **k):
        raise AssertionError('numpy RNG used on the seeded path')
    monkeypatch.setattr(api.os, 'urandom', urandom)
    for name in ('default_rng', 'Generator', 'PCG64', 'randint', 'bytes', 'random'):
        monkeypatch.setattr(np.random, name, no_numpy)
    res = eng.prove_batch_seeded(_Params(P, 16), wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring)
    assert (res.status == 0).all()
    assert [len(b) for b in drawn] == [64]
    ok, st = eng.verify_batch_seeded(_Params(P, 16), wl.msg_hash, wl.ring, res.proofs, res.proof_len, samples=5)
    assert list(ok) == [1, 1] and not st.any()
    assert [len(b) for b in drawn] == [64, 64]
    monkeypatch.undo()
    # the first proof is the oracle's under the tape the drawn seed stands for
    pr = OZ.prove_signature_list(po, wl.msg_hash[0].tobytes(), wl.sig[0].tobytes(), wl.pk[0].tobytes(), int(wl.which[0]),
                                 wl.ring_ints(), Tape(ST.prove_tape(drawn[0][:32], 16, _n(5))))
    assert res.proof_bytes(0) == flat.ser_proof(pr)
    hostsim.params_destroy(P)


def test_signature_list_seed_keyword(hostsim):
    eng = api.Engine.__new__(api.Engine)
    eng.lib, eng.proof_group = hostsim, hostsim.group
    P, _ = common.make_params(hostsim, 75, 16)
    params = _Params(P, 16)
    wl = synth.Workload(B=1, N=5, seed=75)
    keys = wl.ring_ints()
    args = (params, wl.msg_hash[0].tobytes(), wl.sig[0].tobytes(), wl.pk[0].tobytes(), int(wl.which[0]), keys)
    seed = bytes(_seeds(1, 'kw')[0])
    proof = eng.prove_signature_list(*args, seed=seed)
    assert proof.data == eng.prove_signature_list(*args, tape=hostsim.seed_tape(0, _seeds(1, 'kw'), 5, 16)[0].tobytes()).data
    with pytest.raises(ValueError):
        eng.prove_signature_list(*args, tape=bytes(64), seed=seed)
    with pytest.raises(ValueError):
        eng.prove_signature_list(*args, seed=seed[:31])
    # the verifier's default stays the tape; seed= selects the GPU expansion (20 samples need SecLevel >= 20)
    P80, _ = common.make_params(hostsim, 75, 20)
    p20 = _Params(P80, 20)
    proof20 = eng.prove_signature_list(p20, *args[1:], seed=seed)
    assert eng.verify_signature_list(p20, wl.msg_hash[0].tobytes(), keys, proof20, seed=bytes(32)) is True
    with pytest.raises(ValueError):
        eng.verify_signature_list(p20, wl.msg_hash[0].tobytes(), keys, proof20, tape=bytes(64), seed=bytes(32))
    hostsim.params_destroy(P)
    hostsim.params_destroy(P80)


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_seed_tape_on_gpu_matches_oracle(gpu_engine):
    check_seed_tapes(gpu_engine.lib, [(80, 256, (20, 80)), (16, 17, (5,))])


@pytest.mark.gpu
def test_seed_tape_on_gpu_war_matches_oracle(gpu_engine_war):
    check_seed_tapes(gpu_engine_war.lib, [(80, 6, (20,))])


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check_gpu_seeded_prove(L, B=512, N=256, S=80, seed=81):
    import torch
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    P, po = common.make_params(L, seed, S)
    wl = synth.Workload(B=B, N=N, seed=seed)
    seeds = _seeds(B, f'gpu-{seed}')
    tape = L.seed_tape(0, seeds, N, S)
    ref, rlen, rst = common.run_prove(L, P, wl, tape, S)
    assert (rst == 0).all()
    ps = L.proof_max_len(N, S)
    cfg = L.config()
    try:
        for lanes in (1, 3):
            L.set_option('lanes', lanes)
            for chunk in (None, 128):
                if chunk:
                    L.set_option('chunk', chunk)
                    L.set_option('host_chunk', chunk)
                # host buffers
                proofs, plen, st = run_prove_seeded(L, P, wl, seeds, S)
                assert (st == 0).all() and (plen == rlen).all(), (lanes, chunk)
                for b in range(B):     # (row bytes past a proof's length are padding)
                    assert proofs[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes(), ('host', lanes, chunk, b)
                # device buffers (seeds and outputs on the GPU)
                dp = torch.zeros(B * ps, dtype=torch.uint8, device='cuda')
                dl = torch.zeros(B, dtype=torch.int32, device='cuda')
                ds = torch.zeros(B, dtype=torch.int32, device='cuda')
                dm, dsig, dpk, dw, dr, dseed = (_dev(x) for x in (wl.msg_hash, wl.sig, wl.pk, wl.which.view(np.int32), wl.ring, seeds))
                L.prove_batch_seeded(P, B, dm.data_ptr(), dsig.data_ptr(), dpk.data_ptr(), dw.data_ptr(), dr.data_ptr(), N,
                                     dseed.data_ptr(), dp.data_ptr(), ps, dl.data_ptr(), ds.data_ptr())
                torch.cuda.synchronize()
                assert not ds.cpu().numpy().any()
                assert np.array_equal(dl.cpu().numpy().view(np.uint32), rlen), ('device', lanes, chunk)
                got = dp.cpu().numpy().reshape(B, ps)
                for b in range(B):
                    assert got[b, :rlen[b]].tobytes() == ref[b, :rlen[b]].tobytes(), ('device', lanes, chunk, b)
                L.set_option('chunk', cfg['chunk'])
                L.set_option('host_chunk', 2048)
    finally:
        L.set_option('lanes', cfg['lanes'])
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)
    spots = [0, B - 1]
    if L.group != 'tomEdwards256':     # oracle/cpu restates the tomEdwards256 build: the Python oracle checks war256
        for b in spots:
            pr, _ = common.oracle_proof(po, wl, tape, b)
            assert ref[b, :rlen[b]].tobytes() == flat.ser_proof(pr), b
        L.params_destroy(P)
        return
    # spot rows against oracle/cpu on the expanded tape
    g.build_oracle_cpu()
    cpu = ZkaLib(g.ORACLE_CPU)
    hn, hp = cpu.params_generate(synth.params_rnd(seed))
    Pc = cpu.params_create(hn, hp, S)
    sub = synth.Workload.__new__(synth.Workload)
    sub.B, sub.N = len(spots), N
    sub.msg_hash, sub.sig, sub.pk = wl.msg_hash[spots].copy(), wl.sig[spots].copy(), wl.pk[spots].copy()
    sub.which, sub.ring = wl.which[spots].copy(), wl.ring
    cp, cl, cs = common.run_prove(cpu, Pc, sub, tape[spots].copy(), S)
    assert (cs == 0).all()
    for i, b in enumerate(spots):
        assert cp[i, :cl[i]].tobytes() == ref[b, :rlen[b]].tobytes(), b
    cpu.params_destroy(Pc)
    L.params_destroy(P)


@pytest.mark.gpu
def test_seeded_prove_on_gpu_equals_tape_mode(gpu_engine):
    check_gpu_seeded_prove(gpu_engine.lib)


@pytest.mark.gpu
def test_seeded_prove_on_gpu_war_equals_tape_mode(gpu_engine_war):
    check_gpu_seeded_prove(gpu_engine_war.lib, B=256, N=17, S=16, seed=82)


def check_gpu_seeded_verify(L, B=512, N=256, S=80, seed=83, K=20):
    P, _ = common.make_params(L, seed, S)
    wl = synth.Workload(B=B, N=N, seed=seed)
    proofs, plen, st = run_prove_seeded(L, P, wl, _seeds(B, f'gv-{seed}'), S)
    assert (st == 0).all()
    vseeds = _seeds(B, f'gvs-{seed}')
    vt = L.seed_tape(1, vseeds, N, S, K)

    def both(pr, pl, msg):
        ok1, st1 = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        L.verify_batch_seeded(P, B, msg, wl.ring, N, pr, pr.shape[1], pl, vseeds, K, ok1, st1)
        ok2, st2 = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        L.verify_batch_ex(P, B, msg, wl.ring, N, pr, pr.shape[1], pl, vt, vt.shape[1], ok2, st2, K)
        assert np.array_equal(ok1, ok2) and np.array_equal(st1, st2)
        return ok1, st1
    passed = L.stat('agg_pass')
    ok, st = both(proofs, plen, wl.msg_hash)             # every chunk passes the aggregate check as a whole
    assert ok.all() and not st.any()
    assert L.stat('agg_pass') > passed
    wrong, malformed, other_msg = 7, B - 5, B // 2
    bad = proofs.copy()
    bad[wrong, 300] ^= 1                                  # one wrong proof: its chunk takes the per-proof path
    bad[malformed, 0] = 0x05                              # a malformed row (R's tag byte)
    msg = wl.msg_hash.copy()
    msg[other_msg, 0] ^= 1
    failed = L.stat('agg_fail')
    ok, st = both(bad, plen, msg)
    assert L.stat('agg_fail') > failed
    assert st[malformed] != 0 and not ok[other_msg] and not ok[wrong]
    assert ok[[i for i in range(B) if i not in (wrong, malformed, other_msg)]].all()
    L.params_destroy(P)


@pytest.mark.gpu
def test_seeded_verify_on_gpu_equals_tape_mode(gpu_engine):
    check_gpu_seeded_verify(gpu_engine.lib)


@pytest.mark.gpu
def test_seeded_verify_on_gpu_war_equals_tape_mode(gpu_engine_war):
    check_gpu_seeded_verify(gpu_engine_war.lib, B=128, N=17, S=20, seed=84, K=20)
