"""Self-checked proving (include/zkattest.h, "Self-checked proving"): with zka_set_option(ctx, "self_check", 2) every row of
the six batched proveSignatureList calls that the prover accepted is verified with samples = sec_level before the call
releases it.  Rows that pass are byte-identical to the unchecked call; rows that fail get ZKA_ERR_SELF_CHECK (11), zeroed,
with length 0.  Host simulator (both proof groups) and GPU.
"""
import hashlib
from contextlib import contextmanager

import numpy as np
import pytest

import common
from oracle import flat
from oracle import zkattest as OZ
from oracle.big import Tape
from zkp_ecdsa_b200 import synth
from zkp_ecdsa_b200 import verify_tape as VT

SELF_CHECK = 11
KINDS = ('tape', 'seeded', 'hedged')


def _seeds(rows, tag):
    return np.frombuffer(synth.Drbg(rows, f'self-check-{tag}').bytes(32 * rows), np.uint8).reshape(rows, 32).copy()


class Case:
    """One batch: rows over one ring (N) or over a ring set (sizes, ring_of), with a tape and seeds for every row."""

    def __init__(self, L, S, seed, B, N=None, sizes=None, ring_of=None):
        self.L, self.S, self.B = L, S, B
        self.P, self.po = common.make_params(L, seed, S)
        if sizes is None:
            self.w, self.set, self.N = synth.Workload(B=B, N=N, seed=seed), None, N
            deepest = N
        else:
            self.w = synth.RingsWorkload(B, sizes, ring_of, seed=seed)
            self.set = L.rings_create(np.array(sizes, np.uint32), self.w.keys)
            self.sizes = list(sizes)
            deepest = max(sizes[r] for r in set(ring_of))
        self.pl = L.proof_max_len(deepest, S)
        self.tape = synth.random_tape(B, L.prove_tape_len(deepest, S), seed=seed + 1)
        self.seeds = _seeds(B, str(seed))

    def close(self):
        if self.set is not None:
            self.L.rings_destroy(self.set)
        self.L.params_destroy(self.P)

    def fn(self, kind):
        return {'tape': 'prove_batch', 'seeded': 'prove_batch_seeded', 'hedged': 'prove_batch_hedged'}[kind].replace(
            'prove_batch', 'prove_batch_rings' if self.set is not None else 'prove_batch')

    def run(self, kind, dev=False, deterministic=False):
        """(proofs, proof_len, status) of one call, host or device buffers"""
        L, w, B, pl = self.L, self.w, self.B, self.pl
        rnd = self.tape if kind == 'tape' else None if deterministic else self.seeds
        if dev:
            import torch
            keep = []

            def put(a):
                if a is None:
                    return None
                t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
                keep.append(t)
                return t.data_ptr()
            proofs = torch.zeros(B * pl, dtype=torch.uint8, device='cuda')
            plen = torch.zeros(B, dtype=torch.int32, device='cuda')
            st = torch.zeros(B, dtype=torch.int32, device='cuda')
            outs = (proofs.data_ptr(), pl, plen.data_ptr(), st.data_ptr())
        else:
            put = lambda a: a   # noqa: E731
            proofs, plen, st = np.zeros((B, pl), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)
            outs = (proofs, pl, plen, st)
        stmt = tuple(put(a) for a in (w.msg_hash, w.sig, w.pk, w.which))
        rnd_args = (put(rnd), rnd.shape[1]) if kind == 'tape' else (put(rnd),)
        if self.set is None:
            getattr(L, self.fn(kind))(self.P, B, *stmt, put(w.ring), self.N, *rnd_args, *outs)
        else:
            getattr(L, self.fn(kind))(self.P, self.set, put(w.ring_of), B, *stmt, *rnd_args, *outs)
        if dev:
            import torch
            torch.cuda.synchronize()
            return proofs.cpu().numpy().reshape(B, pl), plen.cpu().numpy().view(np.uint32), st.cpu().numpy()
        return proofs, plen, st

    def check_keys(self, kind, deterministic=False):
        """k_b of every row: the caller's seed, the hedged seed, or the first 96 tape bytes"""
        L, w = self.L, self.w
        if kind == 'tape':
            return [self.tape[b, :96].tobytes() for b in range(self.B)]
        seeds = None if deterministic else self.seeds
        if kind == 'seeded':
            k = seeds
        elif self.set is None:
            k = L.hedge_seeds(self.P, self.B, w.msg_hash, w.sig, w.pk, w.which, w.ring, self.N, seeds)
        else:
            k = L.hedge_seeds_rings(self.P, self.set, w.ring_of, self.B, w.msg_hash, w.sig, w.pk, w.which, seeds)
        return [k[b].tobytes() for b in range(self.B)]

    def verify_seeded(self, proofs, plen, seeds):
        """zka_verify_batch[_rings]_seeded with samples = sec_level"""
        L, w, B = self.L, self.w, self.B
        ok, st = np.zeros(B, np.uint8), np.zeros(B, np.int32)
        if self.set is None:
            L.verify_batch_seeded(self.P, B, w.msg_hash, w.ring, self.N, proofs, proofs.shape[1], plen, seeds, self.S, ok, st)
        else:
            L.verify_batch_rings_seeded(self.P, self.set, w.ring_of, B, w.msg_hash, proofs, proofs.shape[1], plen, seeds, self.S,
                                        ok, st)
        return ok, st


def check_seeds(keys):
    """c_b = SHA-256("ZKAttest/check/v1" || k_b)"""
    return np.frombuffer(b''.join(hashlib.sha256(b'ZKAttest/check/v1' + k).digest() for k in keys), np.uint8).reshape(-1, 32).copy()


def rows_equal(a, b):
    (pa, la, sa), (pb, lb, sb) = a, b
    return (np.array_equal(la, lb) and np.array_equal(sa, sb)
            and all(pa[i, :la[i]].tobytes() == pb[i, :lb[i]].tobytes() for i in range(len(la))))


@contextmanager
def self_check(L, on=True):
    L.set_option('self_check', 2 if on else 1)
    try:
        yield
    finally:
        L.set_option('self_check', 1)


@contextmanager
def layout(L, lanes, chunk):
    """lanes and chunk sizes for the duration of a block (chunk None: the defaults)"""
    cfg = L.config()
    try:
        L.set_option('lanes', lanes)
        if chunk:
            L.set_option('chunk', chunk)
            L.set_option('host_chunk', chunk)
        yield
    finally:
        L.set_option('lanes', cfg['lanes'])
        L.set_option('chunk', cfg['chunk'])
        L.set_option('host_chunk', 2048)


def counters(L):
    return L.stat('self_check_rows'), L.stat('self_check_fail')


# ----------------------------------------------------------------------------------- 1. passing rows are unchanged
def check_unchanged(L, case, layouts, devs=(False,)):
    """every call kind, checked and unchecked, over each (lanes, chunk) and buffer kind: identical rows"""
    for kind in KINDS:
        ref = case.run(kind)
        assert not ref[2].any(), (kind, ref[2])
        for lanes, chunk in layouts:
            with layout(L, lanes, chunk):
                for dev in devs:
                    r0, a0 = counters(L), (L.stat('agg_pass'), L.stat('agg_fail'))
                    with self_check(L):
                        got = case.run(kind, dev=dev)
                    assert rows_equal(got, ref), (case.fn(kind), lanes, chunk, dev)
                    assert counters(L) == (r0[0] + case.B, r0[1]), (case.fn(kind), lanes, chunk, dev)
                    assert (L.stat('agg_pass'), L.stat('agg_fail')) == a0      # verify calls only
    # the deterministic hedged call (seeds NULL), twice
    det = case.run('hedged', deterministic=True)
    with self_check(L):
        a = case.run('hedged', deterministic=True)
        b = case.run('hedged', deterministic=True)
    assert not det[2].any() and rows_equal(a, det) and rows_equal(b, det)


MIXED_SIZES = [2, 5, 17, 256]    # depths 1, 3, 5, 8


def mixed_ring_of(B):
    return [i % len(MIXED_SIZES) for i in range(B)]    # depths interleaved row by row


def test_passing_rows_unchanged_hostsim(hostsim):
    L = hostsim
    layouts = ((1, None), (3, 2))                       # one chunk / chunks of 2 rows over three lanes
    case = Case(L, 16, 301, B=5, N=6)
    check_unchanged(L, case, layouts)
    case.close()
    case = Case(L, 16, 302, B=8, sizes=MIXED_SIZES, ring_of=mixed_ring_of(8))
    check_unchanged(L, case, layouts)
    case.close()


def test_passing_rows_unchanged_hostsim_war(hostsim_war):
    L = hostsim_war
    case = Case(L, 16, 303, B=4, N=5)
    check_unchanged(L, case, ((1, None), (3, 2)))
    case.close()
    case = Case(L, 16, 304, B=4, sizes=[3, 9], ring_of=[1, 0, 0, 1])
    check_unchanged(L, case, ((3, 2),))
    case.close()


def test_option_values(hostsim):
    L = hostsim
    r0 = counters(L)
    case = Case(L, 16, 305, B=2, N=5)
    case.run('seeded')                                   # off by default: nothing is checked
    assert counters(L) == r0
    for bad in (0, 3):
        with pytest.raises(Exception):
            L.set_option('self_check', bad)
    case.close()


# ------------------------------------------------------------------------------- 2. a wrong `which` is caught
def wrong_which(case, rows):
    """point rows at a ring entry other than the signer's key (still inside the ring)"""
    w = case.w
    for b in rows:
        size = case.N if case.set is None else case.sizes[int(w.ring_of[b])]
        w.which[b] = (w.which[b] + 1) % size


def check_wrong_which(L, case, bad, kinds=KINDS, devs=(False,), oracle_rows=()):
    wrong_which(case, bad)
    good = [b for b in range(case.B) if b not in bad]
    for kind in kinds:
        off = case.run(kind)
        assert not off[2].any(), (kind, off[2])        # the reference proves them without complaint
        for dev in devs:
            r0 = counters(L)
            with self_check(L):
                on = case.run(kind, dev=dev)
            proofs, plen, st = on
            assert [int(s) for s in st[bad]] == [SELF_CHECK] * len(bad) and not st[good].any(), (kind, dev, st)
            assert not plen[bad].any() and not proofs[bad].any()
            assert rows_equal(tuple(x[good] for x in on), tuple(x[good] for x in off)), (kind, dev)
            assert counters(L) == (r0[0] + case.B, r0[1] + len(bad)), (kind, dev)
        # the rule: the verdict is zka_verify_batch[_rings]_seeded(samples = sec_level, seeds = c) on the unchecked proofs
        ok, vst = case.verify_seeded(off[0], off[1], check_seeds(case.check_keys(kind)))
        assert list(ok == 1) == [b not in bad for b in range(case.B)] and not vst.any(), (kind, ok, vst)
    return off


def oracle_rejects(case, proofs, plen, b):
    """the Python oracle's verifySignatureList (5 samples) on row b of an unchecked call: False"""
    N = case.N
    vt = case.L.seed_tape(1, _seeds(1, f'oracle-{b}'), N, case.S, 5)
    prf = flat.de_proof(proofs[b, :plen[b]].tobytes(), case.S)
    return OZ.verify_signature_list(case.po, case.w.msg_hash[b].tobytes(), case.w.ring_ints(), prf,
                                    Tape(VT.oracle_stream(vt[0].tobytes(), N, case.S)), 5) is False


def check_verify_rejects(case, off, bad):
    """zka_verify_batch (samples 20) rejects the unchecked rows of a wrong `which` and accepts the others"""
    L, w = case.L, case.w
    vts = L.verify_tape_len(case.N, case.S)
    ok, st = common.run_verify(L, case.P, w.msg_hash, w.ring, off[0], off[1], VT.random_verify_tape(case.B, vts, case.N, case.S, seed=9))
    assert list(ok == 1) == [b not in bad for b in range(case.B)] and not st.any(), (ok, st)


def test_wrong_which_hostsim(hostsim):
    L = hostsim
    case = Case(L, 20, 311, B=7, N=6)
    bad = [1, 2, 6]                                     # chunks of 2 over three lanes: both halves of chunk 1, the last row
    with layout(L, 3, 2):
        off = check_wrong_which(L, case, bad)
    check_verify_rejects(case, off, bad)
    assert oracle_rejects(case, off[0], off[1], 1)
    case.close()


def test_wrong_which_rings_hostsim(hostsim):
    L = hostsim
    case = Case(L, 16, 312, B=8, sizes=MIXED_SIZES, ring_of=mixed_ring_of(8))
    with layout(L, 3, 2):
        check_wrong_which(L, case, [0, 3, 5])
    case.close()


def test_wrong_which_hostsim_war(hostsim_war):
    L = hostsim_war
    case = Case(L, 16, 313, B=4, N=5)
    with layout(L, 3, 2):
        check_wrong_which(L, case, [1, 2], kinds=('tape', 'hedged'))
    case.close()


def test_engine_raises_on_failed_check(hostsim):
    from zkp_ecdsa_b200 import api
    L = hostsim
    eng = api.Engine.__new__(api.Engine)
    eng.lib, eng.proof_group = L, L.group
    case = Case(L, 16, 321, B=1, N=5)
    params = type('P', (), {'handle': case.P, 'sec_level': 16})()
    w = case.w
    keys = case.w.ring_ints()
    args = (params, w.msg_hash[0].tobytes(), w.sig[0].tobytes(), w.pk[0].tobytes())
    assert eng.prove_signature_list(*args, int(w.which[0]), keys, seed=bytes(32)).data   # the signer's own index
    other = (int(w.which[0]) + 1) % 5
    eng.prove_signature_list(*args, other, keys, seed=bytes(32))          # unchecked: a proof the verifier rejects
    eng.set_self_check(True)
    try:
        with pytest.raises(api.ZkaProofError) as e:
            eng.prove_signature_list(*args, other, keys, seed=bytes(32))
        assert e.value.status == SELF_CHECK and str(e.value) == 'proof failed its self-check'
        assert eng.prove_signature_list(*args, int(w.which[0]), keys, seed=bytes(32)).data
    finally:
        eng.set_self_check(False)
    case.close()


# ------------------------------------------------------------------------------------------------ 3. precedence
def test_precedence_hostsim(hostsim):
    L = hostsim
    case = Case(L, 16, 331, B=6, N=6)
    w = case.w
    w.pk[1, 40] ^= 1                                    # 1: not a point of the curve
    w.which[2] = 6                                      # 6: inside the padding, outside the ring
    case.tape[3, :32] = 0xff                            # 5: comS1.r >= p256.n
    w.which[4] = (w.which[4] + 1) % 6                   # checked, fails
    off = case.run('tape')
    assert list(off[2]) == [0, 1, 6, 5, 0, 0]
    r0 = counters(L)
    with self_check(L):
        on = case.run('tape')
    assert list(on[2]) == [0, 1, 6, 5, SELF_CHECK, 0]
    assert counters(L) == (r0[0] + 3, r0[1] + 1)        # rows 0, 4 and 5 checked
    keep = [0, 1, 2, 3, 5]
    assert rows_equal(tuple(x[keep] for x in on), tuple(x[keep] for x in off))
    case.close()


# ------------------------------------------------------------------------------------------------ 4. the rule
def test_rule_deterministic_hedged_hostsim(hostsim):
    """c_b of the deterministic hedged call: k_b = the seed derived with seeds NULL"""
    L = hostsim
    case = Case(L, 16, 341, B=3, N=5)
    wrong_which(case, [1])
    off = case.run('hedged', deterministic=True)
    with self_check(L):
        on = case.run('hedged', deterministic=True)
    ok, vst = case.verify_seeded(off[0], off[1], check_seeds(case.check_keys('hedged', deterministic=True)))
    assert list(ok == 1) == list(on[2] != SELF_CHECK) == [True, False, True] and not vst.any()
    case.close()


# ------------------------------------------------------------------------------------------------------------- GPU
def gpu_cases(L, S, seed, B, N, sizes):
    return (Case(L, S, seed, B=B, N=N),
            Case(L, S, seed + 1, B=B, sizes=sizes, ring_of=mixed_ring_of(B) if sizes is MIXED_SIZES
                 else [i % len(sizes) for i in range(B)]))


@pytest.mark.gpu
def test_passing_rows_unchanged_gpu(gpu_engine):
    L = gpu_engine.lib
    for case in gpu_cases(L, 80, 401, 512, 256, MIXED_SIZES):
        check_unchanged(L, case, ((1, None), (3, None), (1, 128), (3, 128)), devs=(False, True))
        case.close()


@pytest.mark.gpu
def test_passing_rows_unchanged_gpu_war(gpu_engine_war):
    L = gpu_engine_war.lib
    for case in gpu_cases(L, 16, 411, 256, 17, [5, 64, 17]):
        check_unchanged(L, case, ((1, None), (3, 64)), devs=(False, True))
        case.close()


@pytest.mark.gpu
def test_wrong_which_gpu(gpu_engine):
    L = gpu_engine.lib
    bad = [0, 127, 128, 255, 256, 300, 511]            # around the boundaries of chunks of 128
    case = Case(L, 80, 421, B=512, N=256)
    with layout(L, 3, 128):
        off = check_wrong_which(L, case, bad, devs=(False, True))
    check_verify_rejects(case, off, bad)
    case.close()
    case = Case(L, 80, 422, B=512, sizes=MIXED_SIZES, ring_of=mixed_ring_of(512))
    with layout(L, 3, 128):
        check_wrong_which(L, case, bad, devs=(False, True))
    case.close()


@pytest.mark.gpu
def test_wrong_which_gpu_war(gpu_engine_war):
    L = gpu_engine_war.lib
    case = Case(L, 16, 431, B=256, N=17)
    with layout(L, 3, 64):
        check_wrong_which(L, case, [0, 63, 64, 200, 255], devs=(False, True))
    case.close()


@pytest.mark.gpu
def test_every_repetition_checked_gpu(gpu_engine):
    """VSampleP256Task belongs to the verifier alone: one checked call runs it on B x sec_level repetitions"""
    L = gpu_engine.lib
    B, S = 1024, 80
    case = Case(L, S, 441, B=B, N=256)
    L.set_profiling(True)
    try:
        for kind in KINDS:
            L.profile_reset()
            case.run(kind, dev=True)
            assert 'VSampleP256Task' not in ''.join(L.profile())   # unchecked: no verifier stage
            L.profile_reset()
            with self_check(L):
                case.run(kind, dev=True)
            items = sum(v['items'] for k, v in L.profile().items() if 'VSampleP256Task' in k)
            assert items == B * S, (kind, items)
    finally:
        L.set_profiling(False)
    case.close()


@pytest.mark.gpu
def test_progress_flags_gpu(gpu_engine):
    """every chunk reported complete holds checked proofs; the rows are those of the unchecked call"""
    L = gpu_engine.lib
    case = Case(L, 80, 451, B=1024, N=256)
    with layout(L, 3, 128):
        ref = case.run('hedged')
        for dev in (True, False):
            nchunks = len(L.chunk_schedule(case.B, not dev)) - 1
            assert nchunks > 3
            flags = np.zeros(nchunks, np.uint32)
            L.set_progress(flags)
            try:
                with self_check(L):
                    got = case.run('hedged', dev=dev)
            finally:
                L.set_progress(None)
            assert flags.all(), (dev, flags)
            assert rows_equal(got, ref), dev
    case.close()
