"""Traceable proofs (include/zkattest.h, "Traceable proofs"), restated on Python ints.

Test infrastructure only, like tests/hedge_rule.py: the device code never reads it.

A traceable proof is the untraced proof followed by a trace block, a sigma proof that (C1, C2) = (k g, x g + k Y) is an
ElGamal encryption "in the exponent" of the signer's key x = keyToInt(pk) under the opener key Y = sk g, and that x is
the value keyXcom = x g + r h commits to:

  C1 = k g    C2 = x g + k Y    A0 = a g + beta h    A1 = c g    A2 = a g + c Y
  e  = SHA-256("ZKAttest/trace/v1" || params digest || Y || msg_hash || proof[0, HEAD_LEN) || C1 C2 A0 A1 A2) mod q
  s_x = a + e x    s_r = beta + e r    s_k = c + e k                                   (mod q)
  block = C1 C2 A0 A1 A2 s_x s_r s_k

The opener recovers D = C2 - sk C1 = x g and the smallest ring index j with (ring[j] mod q) g = D.
"""
from __future__ import annotations

import hashlib
import struct

from oracle import flat
from oracle.seed_tape import P256_P, DOM_PROVE, Stream, rnd

TAG = b'ZKAttest/trace/v1'
DOM_TRACE = 4
Q = P256_P       # order of both proof groups
OK, TAPE_RANGE, IDENTITY_ENC, MALFORMED, TRACE_INVALID, NOT_IN_RING = 0, 5, 7, 9, 12, 13


class TraceError(Exception):
    def __init__(self, status):
        super().__init__(status)
        self.status = status


def trace_len() -> int:
    return 5 * flat.WP + 3 * flat.WS


def params_digest(h_nist: bytes, h_proof: bytes, sec_level: int) -> bytes:
    """The digest zka_params_create computes (include/zkattest.h, "Hedged seeds")."""
    name = flat.PROOF_GROUP.name.encode().ljust(16, b'\0')
    return hashlib.sha256(b'ZKAttest/hedge/params/v1' + name + h_nist + h_proof + struct.pack('<I', sec_level)).digest()


def _g():
    return flat.PROOF_GROUP


def _mul(pt, k):
    return pt.mul(_g().new_scalar(k))


def pubkey(sk: int) -> bytes:
    return _g().generator().mul(_g().new_scalar(sk)).to_bytes()


def _enc(pt) -> bytes:
    b = pt.to_bytes()
    if len(b) != flat.WP:          # the war256 identity has no encoding in a fixed slot
        raise TraceError(IDENTITY_ENC)
    return b


def _sc(v: int) -> bytes:
    return (v % Q).to_bytes(flat.WS, 'big')


def challenge(digest: bytes, Y: bytes, msg_hash: bytes, head: bytes, pts) -> int:
    h = hashlib.sha256(TAG + digest + Y + msg_hash + head[:flat.HEAD_LEN] + b''.join(pts))
    return int.from_bytes(h.digest(), 'big') % Q


def tape_draws(tape_row: bytes, L: int):
    """(r, [k, a, beta, c]) of a tape row: draw 1 and the 32-byte draws at [L, L + 128)."""
    r = int.from_bytes(tape_row[32:64], 'big')
    d = [int.from_bytes(tape_row[L + 32 * t:L + 32 * t + 32], 'big') for t in range(4)]
    return r, d


def seed_draws(seed: bytes):
    """(r, [k, a, beta, c]) of a seeded row: draw 1 on stream(seed, 1, 1) and draw t on stream(seed, 4, t), mod q."""
    return rnd(Stream(seed, DOM_PROVE, 1), Q), [rnd(Stream(seed, DOM_TRACE, t), Q) for t in range(4)]


def prove_block(digest: bytes, h_proof: bytes, Y: bytes, msg_hash: bytes, head: bytes, x: int, r: int, draws) -> bytes:
    """The trace block of one row (raises TraceError(5) / (7))."""
    if any(v >= Q for v in draws):
        raise TraceError(TAPE_RANGE)
    k, a, beta, c = draws
    g = _g()
    G, H, Yp = g.generator(), g.deserialize_point(h_proof), g.deserialize_point(Y)
    pts = [_mul(G, k), _mul(G, x).add(_mul(Yp, k)), _mul(G, a).add(_mul(H, beta)), _mul(G, c), _mul(G, a).add(_mul(Yp, c))]
    enc = [_enc(p) for p in pts]
    e = challenge(digest, Y, msg_hash, head, enc)
    return b''.join(enc) + _sc(a + e * x) + _sc(beta + e * r) + _sc(c + e * k)


def parse_block(block: bytes):
    """(points, scalars) or ValueError, with the base parser's rules."""
    if len(block) != trace_len():
        raise ValueError('trace block length')
    g, WP, WS = _g(), flat.WP, flat.WS
    pts = [g.deserialize_point(block[i * WP:(i + 1) * WP]) for i in range(5)]
    scs = [g.deserialize_scalar(block[5 * WP + i * WS:5 * WP + (i + 1) * WS]).k for i in range(3)]
    return pts, scs


def relations_hold(digest: bytes, h_proof: bytes, Y: bytes, msg_hash: bytes, head: bytes, block: bytes, parsed) -> bool:
    pts, (sx, sr, sk_) = parsed
    C1, C2, A0, A1, A2 = pts
    g = _g()
    G, H, Yp = g.generator(), g.deserialize_point(h_proof), g.deserialize_point(Y)
    kx = g.deserialize_point(head[2 * flat.NP:2 * flat.NP + flat.WP])
    e = challenge(digest, Y, msg_hash, head, [block[i * flat.WP:(i + 1) * flat.WP] for i in range(5)])
    return (_mul(G, sx).add(_mul(H, sr)).eq(A0.add(_mul(kx, e)))
            and _mul(G, sk_).eq(A1.add(_mul(C1, e)))
            and _mul(G, sx).add(_mul(Yp, sk_)).eq(A2.add(_mul(C2, e))))


def verify_row(digest, h_proof, Y, msg_hash, proof: bytes, base_verdict):
    """(ok, status) of a traced row; base_verdict(base_bytes) -> (ok, status) of the untraced verifier."""
    T = trace_len()
    if len(proof) < T:
        return 0, MALFORMED
    block = proof[len(proof) - T:]
    try:
        parsed = parse_block(block)
    except ValueError:
        return 0, MALFORMED
    ok, st = base_verdict(proof[:len(proof) - T])
    if st or not ok:
        return 0, st
    return (1 if relations_hold(digest, h_proof, Y, msg_hash, proof, block, parsed) else 0), 0


def open_row(digest, h_proof, Y, sk: int, msg_hash: bytes, proof: bytes, ring_ints, N: int):
    """(index, status) of zka_open_batch on one row."""
    T = trace_len()
    if len(proof) < T:
        return 0xFFFFFFFF, MALFORMED
    block = proof[len(proof) - T:]
    try:
        parsed = parse_block(block)
    except ValueError:
        return 0xFFFFFFFF, MALFORMED
    if not relations_hold(digest, h_proof, Y, msg_hash, proof, block, parsed):
        return 0xFFFFFFFF, TRACE_INVALID
    C1, C2 = parsed[0][0], parsed[0][1]
    D = C2.sub(_mul(C1, sk)).to_bytes()
    G = _g().generator()
    for j in range(N):
        if _mul(G, ring_ints[j] % Q).to_bytes() == D:
            return j, OK
    return 0xFFFFFFFF, NOT_IN_RING
