"""The ends of the fixed-base commitment walks: a walk starts at the entry of its first window (no addition to the
identity) and, when only the normaliser reads the result, its last addition keeps E, F, G, H instead of the point.
Commitments whose first window holds a zero, +-1 or the half-range digit, whose last window is zero, and the edge values
0, 1 and q - 1 of value and blinder are compared with the oracle's v*g + r*h, on both proof groups.  The split item walks
(g-part, then r*h) and the T1x / T1y affine pairs they feed are covered by a proof of many zero-bit repetitions."""
import pytest

import common
from zkp_ecdsa_b200 import synth


def walk_scalars(q, w, seed):
    """(values, blinders) around the two ends of a walk with w-bit signed windows."""
    nwin = (256 + w) // w
    half = 1 << (w - 1)
    d = synth.Drbg(seed, 'walk-ends')
    hi = lambda: d.below(q >> w) << w   # noqa: E731  (random high part, first window 0)
    # first window digits 0, +1, -1, +2^(w-1), -(2^(w-1) - 1) (a first window has no carry in)
    firsts = [hi(), hi() + 1, hi() + (1 << w) - 1, hi() + half, hi() + half + 1]
    firsts = [v % q for v in firsts]
    # last window zero: values below 2^(w (nwin - 1) - 1) carry nothing into it
    lasts = [d.below(1 << (w * (nwin - 1) - 1)) for _ in range(2)] + [1, half]
    edges = [0, 1, q - 1]
    vs, rs = [], []
    for v in firsts + lasts + edges:
        for r in (edges + firsts[:3] + lasts[:1]):
            vs.append(v)
            rs.append(r)
    return vs, rs


def check_walk_ends(L, seed, sec_level=80):
    w = L.config()['tom_w']
    P, po = common.make_params(L, seed, sec_level)
    g = common.pg(L)
    vs, rs = walk_scalars(g.order, w, seed)
    out = L.tom_commit_batch(P, common.be(vs, 32), common.be(rs, 32))
    for i, (v, r) in enumerate(zip(vs, rs)):
        e = po.ProofGroup.h.dblmul(g.new_scalar(r), po.ProofGroup.g, g.new_scalar(v)).to_bytes()
        if len(e) == 1:
            e = bytes(getattr(L, 'wp', 67))
        assert out[i].tobytes() == e, (i, hex(v), hex(r))
    L.params_destroy(P)


def test_walk_ends_host(hostsim):
    check_walk_ends(hostsim, seed=61)


def test_walk_ends_host_war256(hostsim_war):
    check_walk_ends(hostsim_war, seed=62, sec_level=16)


def test_item_walks_and_affine_pairs_host(hostsim):
    # edge tapes draw 0, 1 and q - 1 into the item secrets and blinders; N = 5 keeps the proof small
    common.check_prove_parity(hostsim, B=2, N=5, seed=63, sec_level=16, make_tape=synth.edge_tape)


@pytest.mark.gpu
def test_walk_ends_device(gpu_engine):
    check_walk_ends(gpu_engine.lib, seed=64)


@pytest.mark.gpu
def test_walk_ends_device_war256(gpu_engine_war):
    check_walk_ends(gpu_engine_war.lib, seed=65, sec_level=16)


@pytest.mark.gpu
def test_item_walks_and_affine_pairs_device(gpu_engine):
    common.check_prove_parity(gpu_engine.lib, B=4, N=9, seed=66, sec_level=16, make_tape=synth.edge_tape)
