"""Argument checks of the batched prove / verify entry points, one fault per call, on the host simulators of both groups.

Every fault is refused before any work: the call returns its code, leaves the outputs untouched and sets
zka_last_error where the library gives a message (elsewhere the previous message stays).  B = 0 returns 0.
"""
import ctypes as C

import numpy as np
import pytest

from zkp_ecdsa_b200 import synth

ARG = -1
RING = 'ring size must be in [2, 2^20]'
PSTRIDE = 'proof_stride < zka_proof_max_len'
PTAPE = 'tape_stride too small'
VTAPE = 'tape_stride < zka_verify_tape_len'
K0 = 'samples must be >= 1'
KS = 'security level not achieved'
RING_OF = 'ring_of[i] >= number of rings in the set'
SENTINEL = 'sec_level must be in [1,80]'   # set by a refused zka_seed_tape before every fault

B, N, S, K = 3, 6, 20, 5                   # one ring of 6: n = 3
SIZES, ROWS = [5, 17], [0, 1, 0]           # a set whose runs have depths 3 | 5 | 3: the first run needs less than the deepest

PROVE = {
    'zka_prove_batch': 'ctx P B msg_hash sig pk which ring N tape tape_stride proofs proof_stride proof_len status',
    'zka_prove_batch_seeded': 'ctx P B msg_hash sig pk which ring N seeds proofs proof_stride proof_len status',
    'zka_prove_batch_rings': 'ctx P rings ring_of B msg_hash sig pk which tape tape_stride proofs proof_stride proof_len status',
    'zka_prove_batch_rings_seeded': 'ctx P rings ring_of B msg_hash sig pk which seeds proofs proof_stride proof_len status',
    'zka_prove_exp_batch': 'ctx P B base s pk q tape tape_stride proofs proof_stride proof_len status',
}
VERIFY = {
    'zka_verify_batch': 'ctx P B msg_hash ring N proofs proof_stride proof_len tape tape_stride ok status',
    'zka_verify_batch_ex': 'ctx P B msg_hash ring N proofs proof_stride proof_len tape tape_stride ok status samples',
    'zka_verify_batch_seeded': 'ctx P B msg_hash ring N proofs proof_stride proof_len seeds samples ok status',
    'zka_verify_batch_rings': 'ctx P rings ring_of B msg_hash proofs proof_stride proof_len tape tape_stride samples ok status',
    'zka_verify_batch_rings_seeded': 'ctx P rings ring_of B msg_hash proofs proof_stride proof_len seeds samples ok status',
    'zka_verify_exp_batch': 'ctx P B base com px py q proofs proof_stride proof_len tape tape_stride samples ok status',
}
OPTIONAL = {'q'}                           # the only pointer an entry point may take as null
SCALARS = {'B', 'N', 'tape_stride', 'proof_stride', 'samples'}


def _faults(name, L, P16):
    """(argument, value, code, message or None) of every one-argument fault that applies to entry point `name`."""
    rings, seeded, exp = 'rings' in name, 'seeded' in name, 'exp' in name
    prove = name.startswith('zka_prove')
    f = []
    if not rings and not exp:
        f += [('N', 1, ARG, RING), ('N', (1 << 20) + 1, ARG, RING)]
    if rings:
        f.append(('ring_of', np.array([0, len(SIZES), 0], np.uint32), ARG, RING_OF))
    deep = max(SIZES) if rings else N                            # the largest ring the call uses
    if prove:
        f.append(('proof_stride', S * L.rep0_len - 1 if exp else L.proof_max_len(deep, S) - 1, ARG, PSTRIDE))
        if not seeded:
            n = 0 if exp else (deep - 1).bit_length()
            f.append(('tape_stride', 32 * (3 + 4 * S + (0 if exp else 5 * n)) - 1, ARG, PTAPE))
    else:
        if name == 'zka_verify_batch':
            f.append(('P', P16, ARG, KS))                        # samples = 20 > sec_level 16
        else:
            f += [('samples', 0, ARG, K0), ('samples', S + 1, ARG, KS)]
        if not seeded:
            k = 20 if name == 'zka_verify_batch' else K
            f.append(('tape_stride', (96 + 32 * 25 * k if exp else L.verify_tape_len_ex(deep, S, k)) - 1, ARG, VTAPE))
        if exp:
            f.append(('proof_stride', 0, ARG, None))
    return f


def _values(L, P, rs):
    z = lambda *shape: np.zeros(shape, np.uint8)   # noqa: E731
    ps = L.proof_max_len(max(SIZES), S)
    v = dict(P=P, rings=rs, ring_of=np.array(ROWS, np.uint32), B=B, N=N, msg_hash=z(B, 32), sig=z(B, 64), pk=z(B, 65),
             which=np.zeros(B, np.uint32), ring=z(N, 32), seeds=z(B, 32), base=z(B, 65), s=z(B, 32), q=z(B, 65),
             com=z(B, 65), px=z(B, L.wp), py=z(B, L.wp), samples=K)
    prove = dict(v, tape=z(B, L.prove_tape_len(max(SIZES), S)), proofs=np.full((B, max(ps, S * L.rep0_len)), 77, np.uint8),
                 proof_len=np.full(B, 77, np.uint32), status=np.full(B, 77, np.int32))
    prove['tape_stride'], prove['proof_stride'] = prove['tape'].shape[1], prove['proofs'].shape[1]
    vt = max(L.verify_tape_len_ex(max(SIZES), S, 20), 96 + 32 * 25 * 20)
    verify = dict(v, tape=z(B, vt), tape_stride=vt, proofs=z(B, S * L.rep0_len), proof_len=np.zeros(B, np.uint32),
                  ok=np.full(B, 77, np.uint8), status=np.full(B, 77, np.int32))
    verify['proof_stride'] = verify['proofs'].shape[1]
    return prove, verify


def _arg(name, value):
    if name in SCALARS:
        return value
    if value is None:
        return C.c_void_p(0)
    return C.c_void_p(value.ctypes.data) if isinstance(value, np.ndarray) else value


def check_call_args(L):
    lib, ctx = L.lib, L.ctx
    rnd = synth.params_rnd(7)
    hn, hp = L.params_generate(rnd)
    P, P16 = L.params_create(hn, hp, S), L.params_create(hn, hp, 16)
    keys = np.frombuffer(synth.Drbg(7, 'call-args').bytes(32 * sum(SIZES)), np.uint8).reshape(-1, 32).copy()
    rs = L.rings_create(np.array(SIZES, np.uint32), keys)
    prove, verify = _values(L, P, rs)
    seeds = np.zeros((1, 32), np.uint8)
    tape = np.zeros((1, 4096), np.uint8)
    checked = 0
    for table, vals, outs in ((PROVE, prove, ('proofs', 'proof_len', 'status')), (VERIFY, verify, ('ok', 'status'))):
        before = {o: vals[o].copy() for o in outs}
        for name, sig in table.items():
            params = sig.split()
            fn = getattr(lib, name)
            faults = [(p, None, ARG, None) for p in params if p not in SCALARS | OPTIONAL] + _faults(name, L, P16)
            faults.append(('B', 0, 0, None))
            for arg, value, code, msg in faults:
                assert lib.zka_seed_tape(ctx, 0, 1, C.c_void_p(seeds.ctypes.data), 8, 0, 0, C.c_void_p(tape.ctypes.data),
                                         tape.shape[1]) == ARG
                assert lib.zka_last_error(ctx).decode() == SENTINEL
                call = dict(vals, ctx=ctx)
                call[arg] = value
                rc = fn(*[_arg(p, call[p]) for p in params])
                assert rc == code, (name, arg, value, rc, lib.zka_last_error(ctx))
                assert lib.zka_last_error(ctx).decode() == (msg or SENTINEL), (name, arg, value)
                for o in outs:
                    assert np.array_equal(vals[o], before[o]), (name, arg, o)
                checked += 1
    assert checked > 150
    L.rings_destroy(rs)
    L.params_destroy(P)
    L.params_destroy(P16)


def test_call_args_hostsim(hostsim):
    check_call_args(hostsim)


def test_call_args_hostsim_war(hostsim_war):
    check_call_args(hostsim_war)


@pytest.mark.parametrize('table', [PROVE, VERIFY])
def test_call_arg_tables_name_every_parameter(table):
    """The tables above follow include/zkattest.h: each entry point's parameter count is the header's."""
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'zkattest.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    for name, sig in table.items():
        m = re.search(r'\b' + name + r'\s*\(([^;]*)\)\s*;', hdr)
        assert m, name
        assert len(m.group(1).split(',')) == len(sig.split()), name
