"""Host-side mirror of the reference's public interface for the hot path.

The reference exports (src/index.ts:17-19, src/zkpAttestList.ts):
    generateParamsList(secLevel = 80)                                   :88
    keyToInt(publicKey)                                                 :94
    proveSignatureList(params, msgHash, sigBytes, publicKey, which, keys)  :104
    verifySignatureList(params, msgHash, keys, proof)                   :147
Node/TypeScript is not available in this image, so the host layer above the C ABI is
Python with the same names (snake_case), argument meaning and error behaviour: malformed
input raises `ZkaProofError(message)` with the reference's message, a failed verification
returns False.  `bindings/node/` holds the TypeScript host + node-addon-api shim a
maintainer would compile where node exists (INTEGRATION.md).

All compute happens in libzkattest.so on the GPU; this module only marshals bytes.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import synth
from .capi import STATUS_MESSAGES, ZkaError, ZkaLib

P256_N = synth.P256_N
TOM_ORDER = synth.P256_P


class ZkaProofError(Exception):
    """Mirrors the reference's `throw new Error(...)` sites (status codes in include/zkattest.h)."""

    def __init__(self, status: int):
        self.status = int(status)
        super().__init__(STATUS_MESSAGES.get(int(status), f'status {status}'))


@dataclass
class SystemParametersList:
    """zkpAttestList.ts:65-78: NistGroup = (p256, G, h_nist), ProofGroup = (tomEdwards256 | war256, g, h_proof)."""
    h_nist: bytes     # 65 B
    h_proof: bytes    # 67 B (tomEdwards256) / 65 B (war256)
    sec_level: int
    handle: object = None   # device tables (zka_params*): 7.3 GB of HBM with the default window widths
    _lib: object = None     # the ZkaLib that owns `handle`
    proof_group: str = 'tomEdwards256'   # ProofGroup.name (instances.ts): selects the library build

    def eq(self, o: 'SystemParametersList') -> bool:
        return (self.h_nist == o.h_nist and self.h_proof == o.h_proof and self.sec_level == o.sec_level
                and self.proof_group == o.proof_group)

    def close(self) -> None:
        """Free the device tables of this parameter set (zka_params_destroy); idempotent."""
        if self.handle is not None and self._lib is not None and getattr(self._lib, 'ctx', None):
            self._lib.params_destroy(self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class SignatureProofList:
    """zkpAttestList.ts:29-61 as its flat byte string (layout in include/zkattest.h)."""
    data: bytes

    def eq(self, o: 'SignatureProofList') -> bool:
        return self.data == o.data


@dataclass
class ProveResult:
    proofs: np.ndarray      # [B, stride] uint8
    proof_len: np.ndarray   # [B] uint32
    status: np.ndarray      # [B] int32

    def proof_bytes(self, b: int) -> bytes:
        return self.proofs[b, :int(self.proof_len[b])].tobytes()


class RingSet:
    """R key rings on the device (zka_rings*): a batch call proves / verifies row i against ring ring_of[i]."""

    def __init__(self, handle, lib, sizes: List[int]):
        self.handle = handle
        self._lib = lib
        self.sizes = list(sizes)
        self.depths = [max(1, (s - 1).bit_length()) for s in self.sizes]   # ceil(log2 N_r), N_r >= 2

    def close(self) -> None:
        """Free the device rings (zka_rings_destroy); idempotent."""
        if self.handle is not None and self._lib is not None and getattr(self._lib, 'ctx', None):
            self._lib.rings_destroy(self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def largest(self, ring_of) -> int:
        """Size of the largest ring `ring_of` uses (strides are taken from it)."""
        used = np.unique(np.asarray(ring_of, np.uint32))
        if used.size and int(used[-1]) >= len(self.sizes):
            raise ValueError(f'ring index {int(used[-1])} outside a set of {len(self.sizes)} rings')
        return max((self.sizes[int(r)] for r in used), default=2)


def _keys_to_ring(keys: Sequence[int]) -> np.ndarray:
    out = np.zeros((len(keys), 32), np.uint8)
    for i, k in enumerate(keys):
        # pad() wraps every key in newScalar (gk.ts:77): reduce mod the proof-group order
        out[i] = np.frombuffer((int(k) % TOM_ORDER).to_bytes(32, 'big'), np.uint8)
    return out


class Engine:
    """One GPU context (zka_ctx).  Raises ZkaError when the CUDA library/device is missing.

    `proof_group`: 'tomEdwards256' (libzkattest.so, what generateParamsList builds) or 'war256' (libzkattest_war256.so:
    the same sources built for the other ProofGroup a SystemParametersList may carry, instances.ts:34-41)."""

    def __init__(self, device: int = 0, lib_path: Optional[str] = None, proof_group: str = 'tomEdwards256'):
        chosen = lib_path is None and 'ZKA_LIB' not in os.environ
        if chosen and proof_group != 'tomEdwards256':
            if proof_group != 'war256':
                raise ValueError(f'invalid group name: {proof_group}')      # instances.ts:66
            from .capi import DEFAULT_LIB
            lib_path = os.path.join(os.path.dirname(DEFAULT_LIB), 'libzkattest_war256.so')
        self.lib = ZkaLib(lib_path, device)
        if chosen:
            assert self.lib.group == proof_group, (self.lib.group, proof_group)
        self.proof_group = self.lib.group

    def close(self):
        self.lib.close()

    def set_self_check(self, on: bool) -> None:
        """Verify every proof of the batched proveSignatureList calls over all sec_level repetitions before it is returned
        (include/zkattest.h, "Self-checked proving"); a proof that fails raises ZkaProofError(11) in prove_signature_list
        and has status 11 in the batch calls.  Off by default."""
        self.lib.set_option('self_check', 2 if on else 1)

    # ------------------------------------------------------------------ reference API
    def generate_params_list(self, sec_level: int = 80, rnd: Optional[bytes] = None) -> SystemParametersList:
        """generateParamsList (zkpAttestList.ts:88-92).  `rnd` = the two rnd() draws (64 B)."""
        if rnd is None:
            rnd = _rnd_below(P256_N) + _rnd_below(TOM_ORDER)
        hn, hp = self.lib.params_generate(rnd)
        return self.load_params(hn, hp, sec_level)

    def load_params(self, h_nist: bytes, h_proof: bytes, sec_level: int = 80) -> SystemParametersList:
        h = self.lib.params_create(h_nist, h_proof, sec_level)
        return SystemParametersList(bytes(h_nist), bytes(h_proof), sec_level, h, self.lib, self.lib.group)

    def key_to_int(self, public_key: bytes) -> int:
        """keyToInt (zkpAttestList.ts:94-102) on the raw 65-byte key (WebCrypto exportKey('raw'))."""
        x, st = self.lib.key_to_int(np.frombuffer(public_key, np.uint8).reshape(1, 65).copy())
        if st[0]:
            raise ZkaProofError(st[0])
        return int.from_bytes(x[0].tobytes(), 'big')

    def prove_signature_list(self, params: SystemParametersList, msg_hash: bytes, sig_bytes: bytes,
                             public_key: bytes, which: int, keys: Sequence[int],
                             tape: Optional[bytes] = None, seed: Optional[bytes] = None) -> SignatureProofList:
        """proveSignatureList (zkpAttestList.ts:104-145); `tape` replaces crypto.getRandomValues, or `seed` (32 secret,
        never reused bytes, include/zkattest.h) has the GPU expand it.  Default: an OS-CSPRNG tape."""
        ring = _keys_to_ring(keys)
        if seed is not None:
            if tape is not None:
                raise ValueError('give either tape or seed')
            res = self.prove_batch_seeded(params, np.frombuffer(msg_hash, np.uint8).reshape(1, 32).copy(),
                                          np.frombuffer(sig_bytes, np.uint8).reshape(1, 64).copy(),
                                          np.frombuffer(public_key, np.uint8).reshape(1, 65).copy(),
                                          np.array([which], np.uint32), ring, _seed_rows(seed, 1))
            if res.status[0]:
                raise ZkaProofError(res.status[0])
            return SignatureProofList(res.proof_bytes(0))
        ts = self.lib.prove_tape_len(len(keys), params.sec_level)
        if tape is None:
            t = synth_os_tape(1, ts, params.sec_level)
        else:
            t = np.zeros((1, ts), np.uint8)
            t[0, :min(ts, len(tape))] = np.frombuffer(tape[:ts], np.uint8)
        res = self.prove_batch(params, np.frombuffer(msg_hash, np.uint8).reshape(1, 32).copy(),
                               np.frombuffer(sig_bytes, np.uint8).reshape(1, 64).copy(),
                               np.frombuffer(public_key, np.uint8).reshape(1, 65).copy(),
                               np.array([which], np.uint32), ring, t)
        if res.status[0]:
            raise ZkaProofError(res.status[0])
        return SignatureProofList(res.proof_bytes(0))

    def verify_signature_list(self, params: SystemParametersList, msg_hash: bytes, keys: Sequence[int],
                              proof: SignatureProofList, tape: Optional[bytes] = None, seed: Optional[bytes] = None) -> bool:
        """verifySignatureList (zkpAttestList.ts:147-184): True/False, raises on malformed input.  `tape` or `seed` (32
        bytes the GPU expands into the verifier's randomness) replace the default OS-CSPRNG tape."""
        if seed is not None and tape is not None:
            raise ValueError('give either tape or seed')
        ring = _keys_to_ring(keys)
        stride = max(len(proof.data), 1)
        pr = np.frombuffer(proof.data, np.uint8).reshape(1, stride).copy()
        msg = np.frombuffer(msg_hash, np.uint8).reshape(1, 32).copy()
        plen = np.array([len(proof.data)], np.uint32)
        if seed is not None:
            ok, st = self.verify_batch_seeded(params, msg, ring, pr, plen, _seed_rows(seed, 1))
        else:
            ts = self.lib.verify_tape_len(len(keys), params.sec_level)
            if tape is None:
                t = synth_os_verify_tape(1, ts, len(keys), params.sec_level)
            else:
                t = np.zeros((1, ts), np.uint8)
                t[0, :min(ts, len(tape))] = np.frombuffer(tape[:ts], np.uint8)
            ok, st = self.verify_batch(params, msg, ring, pr, plen, t)
        if st[0]:
            raise ZkaProofError(st[0])
        return bool(ok[0])

    # ------------------------------------------------------------------ batch variants (additive)
    def prove_batch(self, params, msg_hash, sig, pk, which, ring, tape, proofs=None) -> ProveResult:
        B = msg_hash.shape[0]
        N = ring.shape[0]
        stride = self.lib.proof_max_len(N, params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch(params.handle, B, msg_hash, sig, pk, which, ring, N, tape, tape.shape[1], proofs,
                             proofs.shape[1], plen, status)
        return ProveResult(proofs, plen, status)

    def verify_batch(self, params, msg_hash, ring, proofs, proof_len, tape):
        B = msg_hash.shape[0]
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch(params.handle, B, msg_hash, ring, ring.shape[0], proofs, proofs.shape[1], proof_len,
                              tape, tape.shape[1], ok, status)
        return ok, status

    def prove_batch_seeded(self, params, msg_hash, sig, pk, which, ring, seeds=None, proofs=None) -> ProveResult:
        """prove_batch with the randomness expanded on the GPU from `seeds` (B x 32 uint8, secret, one fresh seed per
        proof; include/zkattest.h).  Default: os.urandom(32 * B)."""
        B = msg_hash.shape[0]
        N = ring.shape[0]
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        stride = self.lib.proof_max_len(N, params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch_seeded(params.handle, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proofs.shape[1], plen,
                                    status)
        return ProveResult(proofs, plen, status)

    def verify_batch_seeded(self, params, msg_hash, ring, proofs, proof_len, seeds=None, samples: int = 20):
        """verify_batch (`samples` sampled repetitions, 20 in verifySignatureList) with the randomness expanded on the
        GPU from `seeds` (B x 32 uint8).  Default: os.urandom(32 * B)."""
        B = msg_hash.shape[0]
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch_seeded(params.handle, B, msg_hash, ring, ring.shape[0], proofs, proofs.shape[1], proof_len, seeds,
                                     samples, ok, status)
        return ok, status

    def _hedge_seeds_arg(self, B, seeds, deterministic):
        if deterministic:
            if seeds is not None:
                raise ValueError('give either seeds or deterministic=True')
            return None
        return _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds

    def prove_batch_hedged(self, params, msg_hash, sig, pk, which, ring, seeds=None, deterministic: bool = False,
                           proofs=None) -> ProveResult:
        """prove_batch_seeded with each row's seed derived on the GPU from `seeds`, the statement and the signature
        (include/zkattest.h, "Hedged seeds"): a repeated seed no longer deanonymises the signer.  Default: os.urandom(32 * B);
        deterministic=True passes no seeds (the randomness then rests on the secrecy of the signature alone)."""
        B = msg_hash.shape[0]
        N = ring.shape[0]
        seeds = self._hedge_seeds_arg(B, seeds, deterministic)
        stride = self.lib.proof_max_len(N, params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch_hedged(params.handle, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proofs.shape[1], plen, status)
        return ProveResult(proofs, plen, status)

    def hedge_seeds(self, params, msg_hash, sig, pk, which, ring, seeds=None, deterministic: bool = False) -> np.ndarray:
        """The B x 32 seeds prove_batch_hedged derives from the same arguments (as secret as the witness; an audit hook).
        With seeds=None and deterministic=False a fresh os.urandom draw is used, as prove_batch_hedged would."""
        B = msg_hash.shape[0]
        seeds = self._hedge_seeds_arg(B, seeds, deterministic)
        return self.lib.hedge_seeds(params.handle, B, msg_hash, sig, pk, which, ring, ring.shape[0], seeds)

    # ------------------------------------------------------------------ ring sets: one batch, many rings
    def load_rings(self, rings: Sequence) -> RingSet:
        """Upload R rings (each a sequence of ints, like `keys`, or an N x 32 uint8 array of entries) as one device set.
        Integer entries are reduced mod the proof-group order like _keys_to_ring; array entries are taken as given (the
        library reduces them the same way)."""
        parts = [np.ascontiguousarray(r, np.uint8).reshape(-1, 32) if isinstance(r, np.ndarray) else _keys_to_ring(r)
                 for r in rings]
        sizes = np.array([p.shape[0] for p in parts], np.uint32)
        keys = np.concatenate(parts, axis=0) if parts else np.zeros((0, 32), np.uint8)
        return RingSet(self.lib.rings_create(sizes, keys), self.lib, [int(s) for s in sizes])

    def prove_batch_rings(self, params, rings: RingSet, ring_of, msg_hash, sig, pk, which, tape, proofs=None) -> ProveResult:
        """prove_batch with row i against ring ring_of[i] of `rings`; tape rows as wide as the largest ring used needs.
        Rows go in any order (rings.depths need not be grouped): the call is one pass of the pipeline."""
        B = msg_hash.shape[0]
        ring_of = np.ascontiguousarray(ring_of, np.uint32)
        stride = self.lib.proof_max_len(rings.largest(ring_of), params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch_rings(params.handle, rings.handle, ring_of, B, msg_hash, sig, pk, which, tape, tape.shape[1], proofs,
                                   proofs.shape[1], plen, status)
        return ProveResult(proofs, plen, status)

    def prove_batch_rings_seeded(self, params, rings: RingSet, ring_of, msg_hash, sig, pk, which, seeds=None,
                                 proofs=None) -> ProveResult:
        """prove_batch_rings with the randomness expanded on the GPU from `seeds` (B x 32).  Default: os.urandom(32 * B)."""
        B = msg_hash.shape[0]
        ring_of = np.ascontiguousarray(ring_of, np.uint32)
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        stride = self.lib.proof_max_len(rings.largest(ring_of), params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch_rings_seeded(params.handle, rings.handle, ring_of, B, msg_hash, sig, pk, which, seeds, proofs,
                                          proofs.shape[1], plen, status)
        return ProveResult(proofs, plen, status)

    def prove_batch_rings_hedged(self, params, rings: RingSet, ring_of, msg_hash, sig, pk, which, seeds=None,
                                 deterministic: bool = False, proofs=None) -> ProveResult:
        """prove_batch_rings_seeded with hedged seeds (see prove_batch_hedged); row i gets the bytes of the one-ring hedged
        call on ring ring_of[i]."""
        B = msg_hash.shape[0]
        ring_of = np.ascontiguousarray(ring_of, np.uint32)
        seeds = self._hedge_seeds_arg(B, seeds, deterministic)
        stride = self.lib.proof_max_len(rings.largest(ring_of), params.sec_level)
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.prove_batch_rings_hedged(params.handle, rings.handle, ring_of, B, msg_hash, sig, pk, which, seeds, proofs,
                                          proofs.shape[1], plen, status)
        return ProveResult(proofs, plen, status)

    def verify_batch_rings(self, params, rings: RingSet, ring_of, msg_hash, proofs, proof_len, tape, samples: int = 20):
        """verify_batch_ex with row i against ring ring_of[i]; tape rows cover the largest ring used."""
        B = msg_hash.shape[0]
        ring_of = np.ascontiguousarray(ring_of, np.uint32)
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch_rings(params.handle, rings.handle, ring_of, B, msg_hash, proofs, proofs.shape[1], proof_len, tape,
                                    tape.shape[1], samples, ok, status)
        return ok, status

    def verify_batch_rings_seeded(self, params, rings: RingSet, ring_of, msg_hash, proofs, proof_len, seeds=None,
                                  samples: int = 20):
        """verify_batch_rings with the randomness expanded on the GPU from `seeds` (B x 32).  Default: os.urandom(32 * B)."""
        B = msg_hash.shape[0]
        ring_of = np.ascontiguousarray(ring_of, np.uint32)
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch_rings_seeded(params.handle, rings.handle, ring_of, B, msg_hash, proofs, proofs.shape[1], proof_len, seeds,
                                           samples, ok, status)
        return ok, status

    # ------------------------------------------------------------------ traceable proofs (include/zkattest.h)
    def trace_keypair(self, sk: Optional[int] = None):
        """(sk, Y): an opener key sk in [1, q) (default: from the OS CSPRNG) and its public key Y = sk g (point bytes).
        Whoever holds sk can open every traced proof made to Y to its signer's ring index."""
        if sk is None:
            while True:
                sk = int.from_bytes(os.urandom(32), 'big')
                if 0 < sk < TOM_ORDER:
                    break
        return sk, self.lib.trace_pubkey(np.frombuffer(int(sk).to_bytes(32, 'big'), np.uint8).copy())

    def _traced_rows(self, B, N, params, proofs):
        stride = self.lib.proof_max_len(N, params.sec_level) + self.lib.trace_len()
        if proofs is None:
            proofs = np.zeros((B, stride), np.uint8)
        return proofs, np.zeros(B, np.uint32), np.zeros(B, np.int32)

    def prove_batch_traced(self, params, msg_hash, sig, pk, which, ring, tape, Y: bytes, proofs=None) -> ProveResult:
        """prove_batch whose accepted rows also carry a trace block to the opener key Y; tape rows need
        zka_prove_tape_len + 128 bytes (the four trace draws behind the prover's)."""
        B, N = msg_hash.shape[0], ring.shape[0]
        proofs, plen, status = self._traced_rows(B, N, params, proofs)
        self.lib.prove_batch_traced(params.handle, B, msg_hash, sig, pk, which, ring, N, tape, tape.shape[1], proofs, proofs.shape[1],
                                    plen, status, Y)
        return ProveResult(proofs, plen, status)

    def prove_batch_traced_seeded(self, params, msg_hash, sig, pk, which, ring, Y: bytes, seeds=None, proofs=None) -> ProveResult:
        """prove_batch_seeded with trace blocks to the opener key Y.  Default seeds: os.urandom(32 * B)."""
        B, N = msg_hash.shape[0], ring.shape[0]
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        proofs, plen, status = self._traced_rows(B, N, params, proofs)
        self.lib.prove_batch_traced_seeded(params.handle, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proofs.shape[1], plen,
                                           status, Y)
        return ProveResult(proofs, plen, status)

    def verify_batch_traced(self, params, msg_hash, ring, proofs, proof_len, tape, Y: bytes, samples: int = 20):
        """verify_batch_ex of traced rows: the untraced verdict of each row's proof and the check of its trace block."""
        B = msg_hash.shape[0]
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch_traced(params.handle, B, msg_hash, ring, ring.shape[0], proofs, proofs.shape[1], proof_len, tape,
                                     tape.shape[1], ok, status, samples, Y)
        return ok, status

    def verify_batch_traced_seeded(self, params, msg_hash, ring, proofs, proof_len, Y: bytes, seeds=None, samples: int = 20):
        B = msg_hash.shape[0]
        seeds = _seed_rows(os.urandom(32 * B), B) if seeds is None else seeds
        ok = np.zeros(B, np.uint8)
        status = np.zeros(B, np.int32)
        self.lib.verify_batch_traced_seeded(params.handle, B, msg_hash, ring, ring.shape[0], proofs, proofs.shape[1], proof_len, seeds,
                                            samples, ok, status, Y)
        return ok, status

    def open_batch(self, params, sk: int, msg_hash, ring, proofs, proof_len):
        """(index, status) per traced row: the smallest ring index whose key made the proof (status 0), or 0xFFFFFFFF
        with status 9 (block does not parse), 12 (block fails its relations) or 13 (key not in the ring / wrong sk)."""
        B = msg_hash.shape[0]
        index = np.zeros(B, np.uint32)
        status = np.zeros(B, np.int32)
        self.lib.open_batch(params.handle, np.frombuffer(int(sk).to_bytes(32, 'big'), np.uint8).copy(), B, msg_hash, ring,
                            ring.shape[0], proofs, proofs.shape[1], proof_len, index, status)
        return index, status


def _seed_rows(seed: bytes, rows: int) -> np.ndarray:
    if len(seed) != 32 * rows:
        raise ValueError(f'a seed is 32 bytes per proof ({32 * rows} expected, {len(seed)} given)')
    return np.frombuffer(bytes(seed), np.uint8).reshape(rows, 32).copy()


def _rnd_below(m: int) -> bytes:
    """rnd(m) of the reference (big.ts:171-181): 32 fresh CSPRNG bytes, redrawn while >= m."""
    while True:
        v = int.from_bytes(os.urandom(32), 'big')
        if v < m:
            return v.to_bytes(32, 'big')


def synth_os_tape(rows: int, stride: int, sec_level: int = 80) -> np.ndarray:
    """Default prover tape = what crypto.getRandomValues would have produced (big.ts:175): every draw is
    32 bytes of os.urandom, redrawn while >= the modulus of that draw (rnd()'s rejection loop; the modulus
    of draw k depends only on k, synth.draw_modulus).  No numpy generator is involved: the revealed
    (alpha_i, r_i, Tx_i.r, Ty_i.r) of 1-bit repetitions are raw tape draws, so the tape must be a CSPRNG."""
    assert stride % 32 == 0
    nd = stride // 32
    t = np.frombuffer(os.urandom(rows * stride), np.uint8).reshape(rows, nd, 32).copy()
    # both moduli start 0xffffffff...: only draws whose top word is all ones can be out of range (2^-32 each)
    cand = np.argwhere((t[:, :, :4] == 255).all(axis=2))
    for r, k in cand:
        m = synth.draw_modulus(int(k), sec_level)
        while int.from_bytes(t[r, k].tobytes(), 'big') >= m:
            t[r, k] = np.frombuffer(os.urandom(32), np.uint8)
    return t.reshape(rows, stride)


def synth_os_verify_tape(rows: int, stride: int, ring_size: int, sec_level: int = 80) -> np.ndarray:
    """Default verifier tape from the OS CSPRNG: Relation.drain scalars (multimult.ts:168-173) and the
    generateIndices bytes rnd(limit - i) (exp.ts:101-106) via secrets.randbelow.  The modulus of a packed
    exp drain depends on the challenge bits, which the host does not know yet, so every 32-byte draw is
    taken uniformly below 0xffffffff * 2^224 (< p256.n < tom.order): 2^-32 short of rnd()'s range, which
    does not affect the soundness of the random linear combination."""
    import secrets
    from .verify_tape import IDX_PAD, ceil_log2, verify_tape_len
    assert stride % 32 == 0 and stride >= verify_tape_len(ring_size)
    t = np.frombuffer(os.urandom(rows * stride), np.uint8).reshape(rows, stride // 32, 32).copy()
    for r, k in np.argwhere((t[:, :, :4] == 255).all(axis=2)):
        while (t[r, k, :4] == 255).all():
            t[r, k] = np.frombuffer(os.urandom(32), np.uint8)
    t = t.reshape(rows, stride)
    g = 32 * (2 * ceil_log2(ring_size) + 1)
    for r in range(rows):
        for i in range(sec_level - 2):
            t[r, g + i] = secrets.randbelow(sec_level - i)
    t[:, g + sec_level - 2:g + IDX_PAD] = 0
    return t
