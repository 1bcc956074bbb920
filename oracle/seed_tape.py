"""The tape a 32-byte seed stands for (include/zkattest.h, "Seeded randomness"), restated in pure Python.

TEST INFRASTRUCTURE (oracle) — see oracle/__init__.py.

stream(seed, domain, index) is the ChaCha20 keystream (RFC 8439 2.3) keyed by the seed with nonce
le32(domain) || le64(index), blocks 0, 1, 2, ... concatenated.  The prover's draw k is rnd(modulus of draw k)
(big.ts:171-181) on stream(seed, 1, k); the verifier's 32-byte slot t is the first candidate of stream(seed, 2, t)
below p256.n; its index byte i is rnd(S - i) on stream(seed, 3, i).  The results are the structured tapes the tape
API takes: prove_tape() the zka_prove_tape_len layout, verify_tape() the zka_verify_tape_len_ex layout.
"""
from __future__ import annotations

import struct

from .big import byte_len

P256_N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551
P256_P = 0xffffffff00000001000000000000000000000000ffffffffffffffffffffffff   # = tomEdwards256 order
DOM_PROVE, DOM_VERIFY, DOM_INDEX = 1, 2, 3
V_IDX_PAD = 96
_M32 = 0xffffffff


def _qr(x, a, b, c, d):
    x[a] = (x[a] + x[b]) & _M32; x[d] ^= x[a]; x[d] = ((x[d] << 16) | (x[d] >> 16)) & _M32
    x[c] = (x[c] + x[d]) & _M32; x[b] ^= x[c]; x[b] = ((x[b] << 12) | (x[b] >> 20)) & _M32
    x[a] = (x[a] + x[b]) & _M32; x[d] ^= x[a]; x[d] = ((x[d] << 8) | (x[d] >> 24)) & _M32
    x[c] = (x[c] + x[d]) & _M32; x[b] ^= x[c]; x[b] = ((x[b] << 7) | (x[b] >> 25)) & _M32


def chacha20_block(key: bytes, counter: int, nonce: bytes) -> bytes:
    """RFC 8439 2.3: one 64-byte block for a 32-byte key, 32-bit counter and 12-byte nonce."""
    assert len(key) == 32 and len(nonce) == 12
    s = [0x61707865, 0x3320646e, 0x79622d32, 0x6b206574] + list(struct.unpack('<8I', key)) + [counter & _M32] + \
        list(struct.unpack('<3I', nonce))
    x = list(s)
    for _ in range(10):
        _qr(x, 0, 4, 8, 12); _qr(x, 1, 5, 9, 13); _qr(x, 2, 6, 10, 14); _qr(x, 3, 7, 11, 15)
        _qr(x, 0, 5, 10, 15); _qr(x, 1, 6, 11, 12); _qr(x, 2, 7, 8, 13); _qr(x, 3, 4, 9, 14)
    return struct.pack('<16I', *[(x[i] + s[i]) & _M32 for i in range(16)])


class Stream:
    """stream(seed, domain, index) as a byte source with the `fill(n)` interface of oracle.big.Tape."""

    def __init__(self, seed: bytes, domain: int, index: int):
        self.key, self.nonce = bytes(seed), struct.pack('<IQ', domain, index)
        self.buf, self.block = b'', 0

    def fill(self, n: int) -> bytes:
        while len(self.buf) < n:
            self.buf += chacha20_block(self.key, self.block, self.nonce)
            self.block += 1
        out, self.buf = self.buf[:n], self.buf[n:]
        return out


def rnd(src, n: int) -> int:
    """big.ts:171-181: byteLen(n)-byte big-endian candidates from `src` until one is below n."""
    while True:
        v = int.from_bytes(src.fill(byte_len(n)), 'big')
        if v < n:
            return v


def draw_modulus(k: int, sec_level: int) -> int:
    """Modulus of prover draw k (include/zkattest.h tape order): comS1.r, alpha_i, r_i mod p256.n, the rest mod tom.order."""
    if k == 0 or (3 <= k < 3 + 4 * sec_level and (k - 3) % 4 < 2):
        return P256_N
    return P256_P


def prove_draw(seed: bytes, k: int, modulus: int) -> bytes:
    return rnd(Stream(seed, DOM_PROVE, k), modulus).to_bytes(32, 'big')


def prove_tape(seed: bytes, S: int, n: int) -> bytes:
    """All 3 + 44 S + 5 n prover draws (S = SecLevel, n = ceil(log2 ring size)): the zka_prove_tape_len layout."""
    return b''.join(prove_draw(seed, k, draw_modulus(k, S)) for k in range(3 + 44 * S + 5 * n))


def verify_tape(seed: bytes, n: int, S: int, K: int) -> bytes:
    """The verify layout for K sampled repetitions: 2n + 1 GK drains, S - 2 index bytes zero-padded to V_IDX_PAD,
    25 K packed exp drains (zka_verify_tape_len_ex bytes)."""
    g = 2 * n + 1
    slots = [rnd(Stream(seed, DOM_VERIFY, t), P256_N).to_bytes(32, 'big') for t in range(g + 25 * K)]
    idx = bytes(rnd(Stream(seed, DOM_INDEX, i), S - i) for i in range(S - 2))
    return b''.join(slots[:g]) + idx + bytes(V_IDX_PAD - len(idx)) + b''.join(slots[g:])
