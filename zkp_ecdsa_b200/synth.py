"""Deterministic synthetic workloads for tests and bench.py (SURVEY.md 8(d)).

Everything derives from a SHA-256 counter DRBG keyed by (seed, label).  P-256 key generation
and ECDSA signing use the `cryptography` package (OpenSSL) — inputs only, nothing measured.
"""
from __future__ import annotations

import hashlib

import numpy as np

P256_N = 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551
P256_P = 0xffffffff00000001000000000000000000000000ffffffffffffffffffffffff  # == tomEdwards256 order


class Drbg:
    def __init__(self, seed: int, label: str):
        self.key = hashlib.sha256(f'zkattest-synth|{seed}|{label}'.encode()).digest()
        self.ctr = 0

    def bytes(self, n: int) -> bytes:
        out = bytearray()
        while len(out) < n:
            out += hashlib.sha256(self.key + self.ctr.to_bytes(8, 'big')).digest()
            self.ctr += 1
        return bytes(out[:n])

    def below(self, m: int) -> int:
        while True:
            v = int.from_bytes(self.bytes(32), 'big')
            if v < m:
                return v


def draw_modulus(k: int, sec_level: int = 80) -> int:
    """Modulus of prover tape draw k (depends only on k; include/zkattest.h)."""
    if k == 0:
        return P256_N
    if k < 3:
        return P256_P
    if k < 3 + 4 * sec_level:
        return P256_N if ((k - 3) % 4) < 2 else P256_P
    return P256_P


def filter_prove_tape(raw: bytes, ndraws: int, sec_level: int = 80) -> bytes:
    """Host-side rnd() rejection loop (big.ts:171-181): consume 32-byte candidates from `raw`
    in order, dropping those >= the modulus of the draw they would feed."""
    out = bytearray()
    pos = 0
    for k in range(ndraws):
        m = draw_modulus(k, sec_level)
        while True:
            cand = raw[pos:pos + 32]
            if len(cand) < 32:
                raise ValueError('raw tape exhausted')
            pos += 32
            if int.from_bytes(cand, 'big') < m:
                out += cand
                break
    return bytes(out)


def random_tape(rows: int, stride: int, seed: int) -> np.ndarray:
    """`rows` tapes of `stride` bytes (multiple of 32) of uniform 32-byte draws, each forced below
    0xffffffff00000000... (< p256.n < p256.p) by resampling the top word (probability 2^-32)."""
    assert stride % 32 == 0
    rng = np.random.Generator(np.random.PCG64(seed))
    t = rng.integers(0, 256, size=(rows, stride), dtype=np.uint8)
    top = t.reshape(rows, stride // 32, 32)[:, :, :4]
    bad = (top == 255).all(axis=2)
    if bad.any():
        t.reshape(rows, stride // 32, 32)[bad, 3] = 0xfe
    return t


def edge_scalars(modulus: int) -> list:
    """Non-zero scalars below `modulus` where digit recoders and carry chains go wrong: 1, m-1, m-2, 2^256 - 2^224 (the
    low end of the range random draws never reach), single bits, windows all equal to 2^(w-1) or 2^(w-1) + 1 for the
    table / MSM widths in use (4..22 bits), all-ones runs, alternating bits."""
    v = {1, 2, modulus - 1, modulus - 2, 0xffffffff << 224, (0xffffffff << 224) + 1, (1 << 255) - 1}
    v |= {1 << b for b in range(0, 256, 7)} | {(1 << b) - 1 for b in range(8, 256, 31)}
    for w in (4, 5, 6, 8, 9, 11, 13, 14, 16, 20, 22):
        for base in (1 << (w - 1), (1 << (w - 1)) + 1):
            v.add(sum(base << (w * j) for j in range(256 // w + 1)) & ((1 << 256) - 1))
    v |= {int('55' * 32, 16), int('aa' * 32, 16), int('0f' * 32, 16)}
    return sorted(x for x in v if 0 < x < modulus)


def edge_tape(rows: int, stride: int, seed: int, sec_level: int = 80) -> np.ndarray:
    """A prover tape (layout of random_tape) whose every 32-byte draw is an edge scalar legal for that draw's modulus
    (draw_modulus); rows and draws cycle through the catalogue at different offsets."""
    t = random_tape(rows, stride, seed)
    cats = {m: edge_scalars(m) for m in (P256_N, P256_P)}
    for r in range(rows):
        for k in range(stride // 32):
            c = cats[draw_modulus(k, sec_level)]
            t[r, 32 * k:32 * k + 32] = np.frombuffer(c[(k * 5 + r * 11 + seed) % len(c)].to_bytes(32, 'big'), np.uint8)
    return t


class Workload:
    """B signing instances sharing one ring of N key x-coordinates."""

    def __init__(self, B: int, N: int, seed: int = 0, distinct_signers: int | None = None):
        from cryptography.hazmat.primitives import serialization
        from cryptography.hazmat.primitives.asymmetric import ec
        self.B, self.N, self.seed = B, N, seed
        ns = min(B, N) if distinct_signers is None else min(distinct_signers, B, N)
        d = Drbg(seed, 'signers')
        dn = Drbg(seed, 'nonces')
        sk_ints = [d.below(P256_N - 1) + 1 for _ in range(ns)]

        def pub(k):   # k*G as 65 raw bytes (OpenSSL does the scalar multiplication)
            return ec.derive_private_key(k, ec.SECP256R1()).public_key().public_bytes(
                serialization.Encoding.X962, serialization.PublicFormat.UncompressedPoint)
        pks = [pub(k) for k in sk_ints]
        # ring: signer j sits at slot slot[j]; filler entries are arbitrary 256-bit values
        dr = Drbg(seed, 'ring')
        ring = [dr.bytes(32) for _ in range(N)]
        perm = np.random.Generator(np.random.PCG64(seed + 7)).permutation(N)[:ns]
        for j in range(ns):
            ring[int(perm[j])] = pks[j][1:33]
        self.ring = np.frombuffer(b''.join(ring), np.uint8).reshape(N, 32).copy()
        self.msg_hash = np.zeros((B, 32), np.uint8)
        self.sig = np.zeros((B, 64), np.uint8)
        self.pk = np.zeros((B, 65), np.uint8)
        self.which = np.zeros(B, np.uint32)
        for b in range(B):
            j = b % ns
            msg = b'zkattest-bench-%d' % b
            digest = hashlib.sha256(msg).digest()
            # deterministic ECDSA: nonce from the DRBG (SURVEY.md 8(d)); r = (kG).x mod n, s = (z + r d)/k
            while True:
                k = dn.below(P256_N - 1) + 1
                r = int.from_bytes(pub(k)[1:33], 'big') % P256_N
                s = pow(k, -1, P256_N) * (int.from_bytes(digest, 'big') + r * sk_ints[j]) % P256_N
                if r and s:
                    break
            self.msg_hash[b] = np.frombuffer(digest, np.uint8)
            self.sig[b] = np.frombuffer(r.to_bytes(32, 'big') + s.to_bytes(32, 'big'), np.uint8)
            self.pk[b] = np.frombuffer(pks[j], np.uint8)
            self.which[b] = int(perm[j])

    def ring_ints(self):
        return [int.from_bytes(self.ring[i].tobytes(), 'big') for i in range(self.N)]


def _p256_pub(k: int) -> bytes:
    """k*G as 65 raw bytes (OpenSSL does the scalar multiplication)."""
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric import ec
    return ec.derive_private_key(k, ec.SECP256R1()).public_key().public_bytes(
        serialization.Encoding.X962, serialization.PublicFormat.UncompressedPoint)


class RingsWorkload:
    """B signing instances over a ring set: row b proves membership in ring ring_of[b] of R rings of the given sizes.

    Ring r holds min(rows of r, sizes[r]) signers of its own at DRBG-chosen slots (a partial Fisher-Yates shuffle); the
    rows of ring r cycle through them, so a ring with one row has a signer of its own.  Filler entries are arbitrary
    256-bit values.  `keys` is the rings' entries concatenated in ring order (the layout of zka_rings_create)."""

    def __init__(self, B: int, sizes, ring_of, seed: int = 0):
        self.B, self.seed = B, seed
        self.sizes = [int(s) for s in sizes]
        self.ring_of = np.asarray(ring_of, np.uint32).reshape(B).copy()
        R = len(self.sizes)
        assert R >= 1 and int(self.ring_of.max(initial=0)) < R
        rows_of = [np.flatnonzero(self.ring_of == r) for r in range(R)]
        d = Drbg(seed, 'rings-signers')
        dn = Drbg(seed, 'rings-nonces')
        dr = Drbg(seed, 'rings-fill')
        self.rings = []
        signer = {}                     # (ring, j) -> (secret key, public key, slot)
        for r, N in enumerate(self.sizes):
            ring = [dr.bytes(32) for _ in range(N)]
            slots = list(range(N))
            for j in range(min(len(rows_of[r]), N)):
                i = j + int.from_bytes(d.bytes(8), 'big') % (N - j)   # (below() is for 256-bit moduli)
                slots[j], slots[i] = slots[i], slots[j]
                sk = d.below(P256_N - 1) + 1
                pk = _p256_pub(sk)
                ring[slots[j]] = pk[1:33]
                signer[r, j] = (sk, pk, slots[j])
            self.rings.append(np.frombuffer(b''.join(ring), np.uint8).reshape(N, 32).copy())
        self.keys = np.concatenate(self.rings, axis=0)
        self.msg_hash = np.zeros((B, 32), np.uint8)
        self.sig = np.zeros((B, 64), np.uint8)
        self.pk = np.zeros((B, 65), np.uint8)
        self.which = np.zeros(B, np.uint32)
        for r in range(R):
            ns = min(len(rows_of[r]), self.sizes[r])
            for j, b in enumerate(rows_of[r]):
                sk, pk, slot = signer[r, j % ns]
                digest = hashlib.sha256(b'zkattest-rings-%d' % b).digest()
                while True:
                    k = dn.below(P256_N - 1) + 1
                    rr = int.from_bytes(_p256_pub(k)[1:33], 'big') % P256_N
                    s = pow(k, -1, P256_N) * (int.from_bytes(digest, 'big') + rr * sk) % P256_N
                    if rr and s:
                        break
                self.msg_hash[b] = np.frombuffer(digest, np.uint8)
                self.sig[b] = np.frombuffer(rr.to_bytes(32, 'big') + s.to_bytes(32, 'big'), np.uint8)
                self.pk[b] = np.frombuffer(pk, np.uint8)
                self.which[b] = slot

    def ring_ints(self, r: int):
        return [int.from_bytes(v.tobytes(), 'big') for v in self.rings[r]]


def params_rnd(seed: int = 0) -> bytes:
    d = Drbg(seed, 'params')
    return d.below(P256_N).to_bytes(32, 'big') + d.below(P256_P).to_bytes(32, 'big')
