"""The hedged seed of a proof (include/zkattest.h, "Hedged seeds"), restated in pure Python with hashlib.

params_digest(), ring_digest() and hedge_seed() derive the 32-byte seed a hedged call feeds to the seeded rule
(oracle/seed_tape.py) from the caller's seed, the statement and the signature.  tests/test_hedged.py checks the
library's kernels (RingDigestTask, SeedHedgeTask) and zka_params_create against them.
"""
from __future__ import annotations

import hashlib
import struct

from oracle.seed_tape import P256_P   # the proof-group order of both groups (tomEdwards256 and war256)

HEDGE_LEAF = 1024


def sha(*parts: bytes) -> bytes:
    return hashlib.sha256(b''.join(parts)).digest()


def params_digest(group: str, h_nist: bytes, h_proof: bytes, sec_level: int) -> bytes:
    """SHA-256("ZKAttest/hedge/params/v1" || group name NUL-padded to 16 || h_nist || h_proof || le32(sec_level))."""
    name = group.encode()
    assert len(name) <= 16 and len(h_nist) == 65
    return sha(b'ZKAttest/hedge/params/v1', name + bytes(16 - len(name)), bytes(h_nist), bytes(h_proof),
               struct.pack('<I', sec_level))


def ring_digest(ring) -> bytes:
    """The digest of a ring of N >= 2 entries (ints or 32-byte big-endian strings): each entry reduced mod the proof-group
    order, padded with entry 0 to 2^n, hashed in leaves of 1024 entries, the leaves under a root."""
    N = len(ring)
    n = (N - 1).bit_length()
    e = [(x if isinstance(x, int) else int.from_bytes(bytes(x), 'big')) % P256_P for x in ring]
    e += [e[0]] * ((1 << n) - N)
    enc = [v.to_bytes(32, 'big') for v in e]
    leaves = [sha(*enc[k:k + HEDGE_LEAF]) for k in range(0, 1 << n, HEDGE_LEAF)]
    return sha(b'ZKAttest/hedge/ring/v1', struct.pack('<II', N, n), *leaves)


def hedge_seed(params_dg: bytes, ring_dg: bytes, seed, msg_hash: bytes, sig: bytes, pk: bytes, which: int) -> bytes:
    """The 32-byte seed of one row of a hedged call; seed None stands for 32 zero bytes (deterministic proofs)."""
    seed = bytes(32) if seed is None else bytes(seed)
    assert len(seed) == 32 and len(msg_hash) == 32 and len(sig) == 64 and len(pk) == 65
    return sha(b'ZKAttest/hedge/prove/v1', params_dg, ring_dg, seed, bytes(msg_hash), bytes(sig), bytes(pk),
               struct.pack('<I', which & 0xffffffff))
