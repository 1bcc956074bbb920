"""Verifier randomness tape helpers (layout in zkp_ecdsa_b200/csrc/zk_verify.cuh / include/zkattest.h)."""
from __future__ import annotations

import numpy as np

V_SAMPLES = 20
IDX_PAD = 96


def ceil_log2(v: int) -> int:
    n = 0
    while (1 << n) < v:
        n += 1
    return n


def verify_tape_len(ring_size: int, samples: int = V_SAMPLES) -> int:
    return 32 * (2 * ceil_log2(ring_size) + 1) + IDX_PAD + 32 * 25 * samples


def random_verify_tape(rows: int, stride: int, ring_size: int, sec_level: int = 80, seed: int = 0) -> np.ndarray:
    """GK drains, 78 (sec_level-2) pre-filtered index bytes, exp drains; all 32-byte draws forced below
    0xffffffff00000000... so they are valid for both moduli (see synth.random_tape)."""
    from .synth import random_tape
    n = ceil_log2(ring_size)
    assert stride >= 32 * (2 * n + 1) + IDX_PAD + 32 and stride % 32 == 0
    t = random_tape(rows, stride, seed)
    g = 32 * (2 * n + 1)
    rng = np.random.Generator(np.random.PCG64(seed + 12345))
    for i in range(sec_level - 2):
        t[:, g + i] = rng.integers(0, sec_level - i, size=rows, dtype=np.uint8)   # rnd(limit - i): uniform < limit - i
    t[:, g + sec_level - 2:g + IDX_PAD] = 0
    return t


def edge_verify_tape(rows: int, stride: int, ring_size: int, sec_level: int = 80, seed: int = 0) -> np.ndarray:
    """random_verify_tape with every 32-byte draw (GK drains and exp drains) replaced by an edge scalar below p256.n,
    legal for both moduli (synth.edge_scalars); the index bytes stay as random_verify_tape makes them."""
    from .synth import P256_N, edge_scalars
    t = random_verify_tape(rows, stride, ring_size, sec_level, seed)
    g = 32 * (2 * ceil_log2(ring_size) + 1)
    cat = edge_scalars(P256_N)
    offs = [o for o in range(0, g, 32)] + [o for o in range(g + IDX_PAD, stride - 31, 32)]
    for r in range(rows):
        for i, o in enumerate(offs):
            t[r, o:o + 32] = np.frombuffer(cat[(i * 3 + r * 13 + seed) % len(cat)].to_bytes(32, 'big'), np.uint8)
    return t


def oracle_stream(tape_row: bytes, ring_size: int, sec_level: int = 80) -> bytes:
    """The byte stream the reference's rnd() calls would consume for this structured tape:
    GK draws, then one byte per generateIndices draw, then the packed 32-byte exp drains."""
    n = ceil_log2(ring_size)
    g = 32 * (2 * n + 1)
    return bytes(tape_row[:g]) + bytes(tape_row[g:g + sec_level - 2]) + bytes(tape_row[g + IDX_PAD:])
