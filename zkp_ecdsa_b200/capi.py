"""ctypes binding of the C ABI in include/zkattest.h (libzkattest.so).

This is the tested surface of the drop-in boundary: the node-addon-api shim of
INTEGRATION.md binds exactly these symbols.  Buffers are numpy uint8 arrays (host) or raw
CUDA device pointers given as ints (e.g. `torch.Tensor.data_ptr()`).

The product library is `zkp_ecdsa_b200/libzkattest.so` (nvcc, sm_90a).  There is no CPU
implementation: `ZkaLib()` raises if the library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, 'libzkattest.so')

SYMBOLS = [
    'zka_init', 'zka_shutdown', 'zka_last_error', 'zka_version', 'zka_launch_count',
    'zka_params_generate', 'zka_params_create', 'zka_params_destroy', 'zka_key_to_int',
    'zka_proof_max_len', 'zka_prove_tape_len', 'zka_verify_tape_len',
    'zka_prove_batch', 'zka_verify_batch',
    'zka_tom_commit_batch', 'zka_p256_mul_batch', 'zka_field_op_batch', 'zka_hash80_batch',
    'zka_get_stream', 'zka_set_profiling', 'zka_profile_reset', 'zka_profile_json', 'zka_config',
    'zka_lanes', 'zka_set_option', 'zka_proofs_pack', 'zka_proofs_unpack', 'zka_verify_batch_ex', 'zka_verify_tape_len_ex',
    'zka_verify_exp_batch', 'zka_verify_membership_batch', 'zka_verify_equality_batch', 'zka_verify_mult_batch',
    'zka_verify_pointadd_batch', 'zka_prove_exp_batch', 'zka_prove_membership_batch',
    'zka_prove_equality_batch', 'zka_prove_mult_batch', 'zka_prove_pointadd_batch', 'zka_stat', 'zka_proof_group', 'zka_set_progress', 'zka_chunk_schedule',
    'zka_prove_batch_seeded', 'zka_verify_batch_seeded', 'zka_seed_tape',
    'zka_rings_create', 'zka_rings_destroy', 'zka_prove_batch_rings', 'zka_prove_batch_rings_seeded', 'zka_verify_batch_rings',
    'zka_verify_batch_rings_seeded', 'zka_prove_batch_hedged', 'zka_prove_batch_rings_hedged', 'zka_hedge_seeds',
    'zka_hedge_seeds_rings', 'zka_trace_len', 'zka_trace_pubkey', 'zka_prove_batch_traced', 'zka_prove_batch_traced_seeded',
    'zka_verify_batch_traced', 'zka_verify_batch_traced_seeded', 'zka_open_batch',
]

STATUS_MESSAGES = {
    0: 'ok',
    1: 'invalid public key',                 # zkpAttestList.ts:117 / weier.ts:83
    2: 'T[i] is at infinity',                # exp.ts:151
    3: 'T1 is at infinity',                  # exp.ts:193
    4: "Points don't add up!",               # pointAdd.ts:105
    5: 'randomness tape draw out of range',
    6: 'index outside the ring',
    7: 'identity point cannot be encoded in a fixed slot',
    8: 'R is at infinity',                   # zkpAttestList.ts:159
    9: 'malformed proof bytes',
    10: 'params not found',                  # exp.ts:270,302
    11: 'proof failed its self-check',       # zka_set_option(ctx, "self_check", 2)
    12: 'trace block fails its relations',   # zka_open_batch
    13: 'traced key is not in the ring',     # zka_open_batch
}


class ZkaError(RuntimeError):
    pass


def _ptr(x):
    """numpy array / bytes / int device pointer / None -> c_void_p"""
    if x is None:
        return C.c_void_p(0)
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        if not x.flags['C_CONTIGUOUS']:
            raise ValueError('array must be C-contiguous')
        return C.c_void_p(x.ctypes.data)
    if isinstance(x, (bytes, bytearray)):
        return C.cast(C.c_char_p(bytes(x)), C.c_void_p)
    raise TypeError(type(x))


class ZkaLib:
    def __init__(self, path: Optional[str] = None, device: int = 0):
        path = path or os.environ.get('ZKA_LIB', DEFAULT_LIB)
        if not os.path.exists(path):
            raise ZkaError(f'{path} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                           '(there is no CPU fallback)')
        self.path = path
        self.lib = C.CDLL(path)
        L = self.lib
        # ProofGroup of this build and its point / scalar sizes in the flat layout (oracle/cpu exports the core ABI only)
        self.group, self.wp, self.ws = 'tomEdwards256', 67, 33
        if hasattr(L, 'zka_proof_group'):
            nm, pb, sb = C.create_string_buffer(32), C.c_int(), C.c_int()
            L.zka_proof_group.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]
            L.zka_proof_group(nm, 32, C.byref(pb), C.byref(sb))
            self.group, self.wp, self.ws = nm.value.decode(), pb.value, sb.value
        self.eq_len = 2 * self.wp + 3 * self.ws                                  # 233 for tomEdwards256
        self.mult_len = 6 * self.wp + 7 * self.ws                                # 633
        self.pa_len = 4 * self.wp + 4 * self.mult_len + 2 * self.eq_len          # 3266
        self.rep0_len = 1 + 65 + 2 * self.wp + 64 + self.pa_len + 2 * self.ws    # 3596
        self.rep1_len = 1 + 65 + 2 * self.wp + 64 + 2 * self.ws                  # 330
        L.zka_init.restype = C.c_int
        L.zka_init.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.zka_shutdown.argtypes = [C.c_void_p]
        L.zka_last_error.restype = C.c_char_p
        L.zka_last_error.argtypes = [C.c_void_p]
        L.zka_launch_count.restype = C.c_uint64
        L.zka_launch_count.argtypes = [C.c_void_p]
        for f in ('zka_proof_max_len', 'zka_prove_tape_len', 'zka_verify_tape_len'):
            getattr(L, f).restype = C.c_size_t
            getattr(L, f).argtypes = [C.c_uint32, C.c_uint32]
        L.zka_params_generate.argtypes = [C.c_void_p] * 4
        L.zka_params_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]
        L.zka_params_destroy.argtypes = [C.c_void_p]
        L.zka_key_to_int.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.zka_prove_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.c_size_t, C.c_void_p, C.c_void_p]
        L.zka_verify_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                       C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_void_p]
        L.zka_tom_commit_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.zka_p256_mul_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.zka_field_op_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.zka_hash80_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.zka_get_stream.restype = C.c_void_p
        L.zka_get_stream.argtypes = [C.c_void_p]
        L.zka_set_profiling.argtypes = [C.c_void_p, C.c_int]
        L.zka_profile_reset.argtypes = [C.c_void_p]
        L.zka_profile_json.restype = C.c_size_t
        L.zka_profile_json.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        L.zka_config.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        if hasattr(L, 'zka_verify_batch_ex') and not hasattr(L, 'zka_set_option'):
            L.zka_verify_tape_len_ex.restype = C.c_size_t
            L.zka_verify_tape_len_ex.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
            L.zka_verify_batch_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32]
        if hasattr(L, 'zka_set_option'):      # (oracle/cpu exports the core ABI only)
            L.zka_lanes.argtypes = [C.c_void_p]
            L.zka_verify_tape_len_ex.restype = C.c_size_t
            L.zka_verify_tape_len_ex.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
            L.zka_verify_batch_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32]
            L.zka_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_long]
            L.zka_stat.restype = C.c_longlong
            L.zka_stat.argtypes = [C.c_void_p, C.c_char_p]
            L.zka_verify_exp_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6 + [C.c_size_t, C.c_void_p, C.c_void_p,
                                               C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p]
            L.zka_verify_membership_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                      C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
            for f in ('zka_verify_equality_batch', 'zka_verify_mult_batch', 'zka_verify_pointadd_batch'):
                getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                          C.c_void_p, C.c_void_p]
            L.zka_prove_exp_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [C.c_size_t, C.c_void_p, C.c_size_t,
                                              C.c_void_p, C.c_void_p]
            L.zka_prove_membership_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                     C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
            for f in ('zka_prove_equality_batch', 'zka_prove_mult_batch'):
                getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                          C.c_void_p]
            L.zka_prove_pointadd_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
            L.zka_proofs_pack.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                          C.c_void_p, C.c_void_p]
            L.zka_proofs_unpack.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p]
        if hasattr(L, 'zka_seed_tape'):
            L.zka_prove_batch_seeded.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p,
                                                 C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
            L.zka_verify_batch_seeded.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                  C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
            L.zka_seed_tape.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                        C.c_size_t]
        if hasattr(L, 'zka_rings_create'):
            L.zka_rings_create.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
            L.zka_rings_destroy.argtypes = [C.c_void_p]
            L.zka_prove_batch_rings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [
                C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
            L.zka_prove_batch_rings_seeded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6 + [
                C.c_size_t, C.c_void_p, C.c_void_p]
            L.zka_verify_batch_rings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                                 C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p]
            L.zka_verify_batch_rings_seeded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                        C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                        C.c_void_p]
        if hasattr(L, 'zka_hedge_seeds'):
            L.zka_prove_batch_hedged.argtypes = L.zka_prove_batch_seeded.argtypes
            L.zka_prove_batch_rings_hedged.argtypes = L.zka_prove_batch_rings_seeded.argtypes
            L.zka_hedge_seeds.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p, C.c_void_p]
            L.zka_hedge_seeds_rings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
        if hasattr(L, 'zka_open_batch'):
            L.zka_trace_len.restype = C.c_size_t
            L.zka_trace_len.argtypes = []
            L.zka_trace_pubkey.argtypes = [C.c_void_p] * 3
            L.zka_prove_batch_traced.argtypes = L.zka_prove_batch.argtypes + [C.c_void_p]
            L.zka_prove_batch_traced_seeded.argtypes = L.zka_prove_batch_seeded.argtypes + [C.c_void_p]
            L.zka_verify_batch_traced.argtypes = L.zka_verify_batch_ex.argtypes + [C.c_void_p]
            L.zka_verify_batch_traced_seeded.argtypes = L.zka_verify_batch_seeded.argtypes + [C.c_void_p]
            L.zka_open_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        ctx = C.c_void_p()
        rc = L.zka_init(device, C.byref(ctx))
        if rc != 0 or not ctx:
            raise ZkaError(f'zka_init(device={device}) failed with {rc}: no usable CUDA device '
                           '(libzkattest has no CPU fallback)')
        self.ctx = ctx
        self.device = device

    # ------------------------------------------------------------------ helpers
    def close(self):
        if getattr(self, 'ctx', None):
            self.lib.zka_shutdown(self.ctx)
            self.ctx = None

    def _check(self, rc, what):
        if rc != 0:
            raise ZkaError(f'{what} failed ({rc}): {self.lib.zka_last_error(self.ctx).decode()}')

    def launch_count(self) -> int:
        return int(self.lib.zka_launch_count(self.ctx))

    def stream_ptr(self) -> int:
        return int(self.lib.zka_get_stream(self.ctx) or 0)

    def set_profiling(self, on: bool):
        self._check(self.lib.zka_set_profiling(self.ctx, 1 if on else 0), 'zka_set_profiling')

    def profile_reset(self):
        self._check(self.lib.zka_profile_reset(self.ctx), 'zka_profile_reset')

    def profile(self) -> dict:
        import json
        n = self.lib.zka_profile_json(self.ctx, None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        self.lib.zka_profile_json(self.ctx, buf, len(buf))
        return json.loads(buf.value.decode())

    def config(self) -> dict:
        w, nw, ch = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.zka_config(self.ctx, C.byref(w), C.byref(nw), C.byref(ch)), 'zka_config')
        lanes = int(self.lib.zka_lanes(self.ctx)) if hasattr(self.lib, 'zka_lanes') else 1
        cfg = {'tom_w': w.value, 'tom_nwin': nw.value, 'chunk': ch.value, 'lanes': lanes}
        # the first tom_n_lo of the tom_nwin windows have tom_w bits, the others tom_w + 1 (ZKA_TOM_NWIN; all of them with
        # ZKA_TOM_W); tom_fallback: the tables asked for did not fit and the context walks one lookup more
        if hasattr(self.lib, 'zka_stat') and self.stat('tom_n_lo') >= 0:
            cfg.update(tom_n_lo=self.stat('tom_n_lo'), tom_fallback=bool(self.stat('tom_fallback')))
        return cfg

    def set_option(self, key: str, value: int):
        self._check(self.lib.zka_set_option(self.ctx, key.encode(), int(value)), f'zka_set_option({key})')

    def chunk_schedule(self, B: int, host_buffers: bool = False):
        """Chunk offsets [0, ..., B] a prove call over B proofs will use (deterministic; the same on every rank)."""
        off = np.zeros(4096, np.uint32)
        self.lib.zka_chunk_schedule.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_uint32]
        n = self.lib.zka_chunk_schedule(self.ctx, B, 1 if host_buffers else 0, _ptr(off), off.size)
        if n < 0:
            raise ZkaError('zka_chunk_schedule')
        return [int(v) for v in off[:n + 1]]

    def set_progress(self, flags: Optional[np.ndarray]):
        """flags[k] (uint32, kept alive by the caller) becomes 1 when chunk k of the running prove call is complete."""
        self.lib.zka_set_progress.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        if flags is None:
            self._check(self.lib.zka_set_progress(self.ctx, None, 0), 'zka_set_progress')
        else:
            assert flags.dtype == np.uint32 and flags.flags['C_CONTIGUOUS']
            self._check(self.lib.zka_set_progress(self.ctx, _ptr(flags), flags.size), 'zka_set_progress')

    def stat(self, key: str) -> int:
        """Counters since zka_init ('agg_pass', 'agg_fail': verifier chunks decided by the chunk-wide aggregate check /
        sent on to the per-proof evaluation)."""
        return int(self.lib.zka_stat(self.ctx, key.encode()))

    def proof_max_len(self, ring_size, sec_level=80): return int(self.lib.zka_proof_max_len(ring_size, sec_level))
    def prove_tape_len(self, ring_size, sec_level=80): return int(self.lib.zka_prove_tape_len(ring_size, sec_level))
    def verify_tape_len(self, ring_size, sec_level=80): return int(self.lib.zka_verify_tape_len(ring_size, sec_level))

    # ------------------------------------------------------------------ params
    def params_generate(self, rnd: bytes):
        assert len(rnd) == 64
        hn = np.zeros(65, np.uint8)
        hp = np.zeros(self.wp, np.uint8)
        self._check(self.lib.zka_params_generate(self.ctx, _ptr(rnd), _ptr(hn), _ptr(hp)), 'zka_params_generate')
        return hn.tobytes(), hp.tobytes()

    def params_create(self, h_nist: bytes, h_proof: bytes, sec_level: int = 80):
        h = C.c_void_p()
        self._check(self.lib.zka_params_create(self.ctx, _ptr(h_nist), _ptr(h_proof), sec_level, C.byref(h)),
                    'zka_params_create')
        return h

    def params_destroy(self, h):
        self.lib.zka_params_destroy(h)

    def key_to_int(self, pk: np.ndarray):
        count = pk.shape[0]
        out = np.zeros((count, 32), np.uint8)
        st = np.zeros(count, np.int32)
        self._check(self.lib.zka_key_to_int(self.ctx, count, _ptr(pk), _ptr(out), _ptr(st)), 'zka_key_to_int')
        return out, st

    # ------------------------------------------------------------------ hot path
    def prove_batch(self, params, B, msg_hash, sig, pk, which, ring, N, tape, tape_stride,
                    proofs, proof_stride, proof_len, status):
        self._check(self.lib.zka_prove_batch(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which),
                                             _ptr(ring), N, _ptr(tape), tape_stride, _ptr(proofs), proof_stride,
                                             _ptr(proof_len), _ptr(status)), 'zka_prove_batch')

    def verify_batch(self, params, B, msg_hash, ring, N, proofs, proof_stride, proof_len, tape, tape_stride,
                     ok, status):
        self._check(self.lib.zka_verify_batch(self.ctx, params, B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs),
                                              proof_stride, _ptr(proof_len), _ptr(tape), tape_stride, _ptr(ok),
                                              _ptr(status)), 'zka_verify_batch')

    def verify_tape_len_ex(self, ring_size, sec_level, samples):
        return int(self.lib.zka_verify_tape_len_ex(ring_size, sec_level, samples))

    def verify_batch_ex(self, params, B, msg_hash, ring, N, proofs, proof_stride, proof_len, tape, tape_stride, ok, status, samples):
        self._check(self.lib.zka_verify_batch_ex(self.ctx, params, B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs), proof_stride,
                                                 _ptr(proof_len), _ptr(tape), tape_stride, _ptr(ok), _ptr(status), samples),
                    'zka_verify_batch_ex')

    # ------------------------------------------------------------------ seeded randomness
    def prove_batch_seeded(self, params, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proof_stride, proof_len, status):
        self._check(self.lib.zka_prove_batch_seeded(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which), _ptr(ring),
                                                    N, _ptr(seeds), _ptr(proofs), proof_stride, _ptr(proof_len), _ptr(status)),
                    'zka_prove_batch_seeded')

    def verify_batch_seeded(self, params, B, msg_hash, ring, N, proofs, proof_stride, proof_len, seeds, samples, ok, status):
        self._check(self.lib.zka_verify_batch_seeded(self.ctx, params, B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs), proof_stride,
                                                     _ptr(proof_len), _ptr(seeds), samples, _ptr(ok), _ptr(status)),
                    'zka_verify_batch_seeded')

    def seed_tape(self, kind, seeds, ring_size, sec_level=80, samples=20) -> np.ndarray:
        """The tape `seeds` (B x 32) stand for: kind 0 the prover's (zka_prove_tape_len), 1 the verifier's for `samples`."""
        B = seeds.shape[0]
        ln = self.prove_tape_len(ring_size, sec_level) if kind == 0 else self.verify_tape_len_ex(ring_size, sec_level, samples)
        out = np.zeros((B, ln), np.uint8)
        self._check(self.lib.zka_seed_tape(self.ctx, kind, B, _ptr(seeds), ring_size, sec_level, samples, _ptr(out), ln),
                    'zka_seed_tape')
        return out

    # ------------------------------------------------------------------ ring sets (row i against ring ring_of[i])
    def rings_create(self, sizes: np.ndarray, keys):
        """sizes: R uint32 (host); keys: sum(sizes) x 32 bytes, host array or device pointer -> zka_rings* handle."""
        h = C.c_void_p()
        self._check(self.lib.zka_rings_create(self.ctx, sizes.size, _ptr(sizes), _ptr(keys), C.byref(h)), 'zka_rings_create')
        return h

    def rings_destroy(self, h):
        self.lib.zka_rings_destroy(h)

    def prove_batch_rings(self, params, rings, ring_of, B, msg_hash, sig, pk, which, tape, tape_stride, proofs, proof_stride,
                          proof_len, status):
        self._check(self.lib.zka_prove_batch_rings(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(sig), _ptr(pk),
                                                   _ptr(which), _ptr(tape), tape_stride, _ptr(proofs), proof_stride, _ptr(proof_len),
                                                   _ptr(status)), 'zka_prove_batch_rings')

    def prove_batch_rings_seeded(self, params, rings, ring_of, B, msg_hash, sig, pk, which, seeds, proofs, proof_stride, proof_len,
                                 status):
        self._check(self.lib.zka_prove_batch_rings_seeded(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(sig), _ptr(pk),
                                                          _ptr(which), _ptr(seeds), _ptr(proofs), proof_stride, _ptr(proof_len),
                                                          _ptr(status)), 'zka_prove_batch_rings_seeded')

    def verify_batch_rings(self, params, rings, ring_of, B, msg_hash, proofs, proof_stride, proof_len, tape, tape_stride, samples, ok,
                           status):
        self._check(self.lib.zka_verify_batch_rings(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(proofs), proof_stride,
                                                    _ptr(proof_len), _ptr(tape), tape_stride, samples, _ptr(ok), _ptr(status)),
                    'zka_verify_batch_rings')

    def verify_batch_rings_seeded(self, params, rings, ring_of, B, msg_hash, proofs, proof_stride, proof_len, seeds, samples, ok,
                                  status):
        self._check(self.lib.zka_verify_batch_rings_seeded(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(proofs),
                                                           proof_stride, _ptr(proof_len), _ptr(seeds), samples, _ptr(ok), _ptr(status)),
                    'zka_verify_batch_rings_seeded')

    # ------------------------------------------------------------------ hedged seeds (seeds may be None: NULL)
    def prove_batch_hedged(self, params, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proof_stride, proof_len, status):
        self._check(self.lib.zka_prove_batch_hedged(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which), _ptr(ring),
                                                    N, _ptr(seeds), _ptr(proofs), proof_stride, _ptr(proof_len), _ptr(status)),
                    'zka_prove_batch_hedged')

    def prove_batch_rings_hedged(self, params, rings, ring_of, B, msg_hash, sig, pk, which, seeds, proofs, proof_stride, proof_len,
                                 status):
        self._check(self.lib.zka_prove_batch_rings_hedged(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(sig), _ptr(pk),
                                                          _ptr(which), _ptr(seeds), _ptr(proofs), proof_stride, _ptr(proof_len),
                                                          _ptr(status)), 'zka_prove_batch_rings_hedged')

    def hedge_seeds(self, params, B, msg_hash, sig, pk, which, ring, N, seeds, out=None) -> np.ndarray:
        """The B x 32 seeds a hedged call derives (as secret as the witness)."""
        out = np.zeros((B, 32), np.uint8) if out is None else out
        self._check(self.lib.zka_hedge_seeds(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which), _ptr(ring), N,
                                             _ptr(seeds), _ptr(out)), 'zka_hedge_seeds')
        return out

    def hedge_seeds_rings(self, params, rings, ring_of, B, msg_hash, sig, pk, which, seeds, out=None) -> np.ndarray:
        out = np.zeros((B, 32), np.uint8) if out is None else out
        self._check(self.lib.zka_hedge_seeds_rings(self.ctx, params, rings, _ptr(ring_of), B, _ptr(msg_hash), _ptr(sig), _ptr(pk),
                                                   _ptr(which), _ptr(seeds), _ptr(out)), 'zka_hedge_seeds_rings')
        return out

    # ------------------------------------------------------------------ traceable proofs (Y: the opener key, point bytes)
    def trace_len(self) -> int:
        return int(self.lib.zka_trace_len())

    def trace_pubkey(self, sk) -> bytes:
        Y = np.zeros(self.wp, np.uint8)
        self._check(self.lib.zka_trace_pubkey(self.ctx, _ptr(sk), _ptr(Y)), 'zka_trace_pubkey')
        return Y.tobytes()

    def prove_batch_traced(self, params, B, msg_hash, sig, pk, which, ring, N, tape, tape_stride, proofs, proof_stride, proof_len,
                           status, Y):
        self._check(self.lib.zka_prove_batch_traced(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which), _ptr(ring),
                                                    N, _ptr(tape), tape_stride, _ptr(proofs), proof_stride, _ptr(proof_len),
                                                    _ptr(status), _ptr(Y)), 'zka_prove_batch_traced')

    def prove_batch_traced_seeded(self, params, B, msg_hash, sig, pk, which, ring, N, seeds, proofs, proof_stride, proof_len, status, Y):
        self._check(self.lib.zka_prove_batch_traced_seeded(self.ctx, params, B, _ptr(msg_hash), _ptr(sig), _ptr(pk), _ptr(which),
                                                           _ptr(ring), N, _ptr(seeds), _ptr(proofs), proof_stride, _ptr(proof_len),
                                                           _ptr(status), _ptr(Y)), 'zka_prove_batch_traced_seeded')

    def verify_batch_traced(self, params, B, msg_hash, ring, N, proofs, proof_stride, proof_len, tape, tape_stride, ok, status, samples,
                            Y):
        self._check(self.lib.zka_verify_batch_traced(self.ctx, params, B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs), proof_stride,
                                                     _ptr(proof_len), _ptr(tape), tape_stride, _ptr(ok), _ptr(status), samples, _ptr(Y)),
                    'zka_verify_batch_traced')

    def verify_batch_traced_seeded(self, params, B, msg_hash, ring, N, proofs, proof_stride, proof_len, seeds, samples, ok, status, Y):
        self._check(self.lib.zka_verify_batch_traced_seeded(self.ctx, params, B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs),
                                                            proof_stride, _ptr(proof_len), _ptr(seeds), samples, _ptr(ok), _ptr(status),
                                                            _ptr(Y)), 'zka_verify_batch_traced_seeded')

    def open_batch(self, params, sk, B, msg_hash, ring, N, proofs, proof_stride, proof_len, index, status):
        self._check(self.lib.zka_open_batch(self.ctx, params, _ptr(sk), B, _ptr(msg_hash), _ptr(ring), N, _ptr(proofs), proof_stride,
                                            _ptr(proof_len), _ptr(index), _ptr(status)), 'zka_open_batch')

    # ------------------------------------------------------------------ stand-alone sub-proof verifiers
    def verify_exp_batch(self, params, base, com, px, py, q, proofs, proof_len, tape, samples):
        B = base.shape[0]
        ok = np.zeros(B, np.uint8)
        st = np.zeros(B, np.int32)
        self._check(self.lib.zka_verify_exp_batch(self.ctx, params, B, _ptr(base), _ptr(com), _ptr(px), _ptr(py), _ptr(q), _ptr(proofs),
                                                  proofs.shape[1], _ptr(proof_len), _ptr(tape), tape.shape[1], samples, _ptr(ok), _ptr(st)),
                    'zka_verify_exp_batch')
        return ok, st

    def verify_membership_batch(self, params, com, ring, proofs, proof_len, tape):
        B = com.shape[0]
        ok = np.zeros(B, np.uint8)
        st = np.zeros(B, np.int32)
        self._check(self.lib.zka_verify_membership_batch(self.ctx, params, B, _ptr(com), _ptr(ring), ring.shape[0], _ptr(proofs),
                                                         proofs.shape[1], _ptr(proof_len), _ptr(tape), tape.shape[1], _ptr(ok), _ptr(st)),
                    'zka_verify_membership_batch')
        return ok, st

    def prove_exp_batch(self, params, base, s, pk, q, tape, sec_level):
        B = base.shape[0]
        stride = sec_level * self.rep0_len
        proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        st = np.zeros(B, np.int32)
        self._check(self.lib.zka_prove_exp_batch(self.ctx, params, B, _ptr(base), _ptr(s), _ptr(pk), _ptr(q), _ptr(tape), tape.shape[1],
                                                 _ptr(proofs), stride, _ptr(plen), _ptr(st)), 'zka_prove_exp_batch')
        return proofs, plen, st

    def prove_membership_batch(self, params, com_r, index, ring, tape):
        B, N = com_r.shape[0], ring.shape[0]
        n = max(1, (N - 1).bit_length()) if N > 1 else 0
        stride = 1 + 4 * n * self.wp + (3 * n + 1) * self.ws
        proofs = np.zeros((B, stride), np.uint8)
        plen = np.zeros(B, np.uint32)
        st = np.zeros(B, np.int32)
        self._check(self.lib.zka_prove_membership_batch(self.ctx, params, B, _ptr(com_r), _ptr(index), _ptr(ring), N, _ptr(tape),
                                                        tape.shape[1], _ptr(proofs), stride, _ptr(plen), _ptr(st)),
                    'zka_prove_membership_batch')
        return proofs, plen, st

    def prove_sub_batch(self, kind: str, params, inputs, tape, blinders=None):
        """kind 'equality' (inputs [B, 3*32]), 'mult' ([B, 6*32]) or 'pointadd' (inputs [B, 3*65] + blinders [B, 6*32])"""
        B = inputs.shape[0]
        nc, plen = {'equality': (2, self.eq_len), 'mult': (3, self.mult_len), 'pointadd': (6, self.pa_len)}[kind]
        com = np.zeros((B, nc * self.wp), np.uint8)
        proofs = np.zeros((B, plen), np.uint8)
        st = np.zeros(B, np.int32)
        if kind == 'pointadd':
            rc = self.lib.zka_prove_pointadd_batch(self.ctx, params, B, _ptr(inputs), _ptr(blinders), _ptr(tape), tape.shape[1], _ptr(com),
                                                   _ptr(proofs), _ptr(st))
        else:
            rc = getattr(self.lib, f'zka_prove_{kind}_batch')(self.ctx, params, B, _ptr(inputs), _ptr(tape), tape.shape[1], _ptr(com),
                                                              _ptr(proofs), _ptr(st))
        self._check(rc, f'zka_prove_{kind}_batch')
        return com, proofs, st

    def verify_sub_batch(self, kind: str, params, points, proofs, tape):
        """kind in {'equality', 'mult', 'pointadd'}; points [B, k*67], proofs [B, 233|633|3266], tape [B, >= 32*draws]"""
        B = points.shape[0]
        ok = np.zeros(B, np.uint8)
        st = np.zeros(B, np.int32)
        fn = getattr(self.lib, f'zka_verify_{kind}_batch')
        self._check(fn(self.ctx, params, B, _ptr(points), _ptr(proofs), _ptr(tape), tape.shape[1], _ptr(ok), _ptr(st)),
                    f'zka_verify_{kind}_batch')
        return ok, st

    # ------------------------------------------------------------------ multi-GPU helpers
    def proofs_pack(self, B, proofs, stride, proof_len, packed, cap, offsets, stream=0):
        self._check(self.lib.zka_proofs_pack(self.ctx, B, _ptr(proofs), stride, _ptr(proof_len), _ptr(packed), cap, _ptr(offsets),
                                             C.c_void_p(stream or 0)), 'zka_proofs_pack')

    def proofs_unpack(self, B, packed, cap, proof_len, proofs, stride, offsets, stream=0):
        self._check(self.lib.zka_proofs_unpack(self.ctx, B, _ptr(packed), cap, _ptr(proof_len), _ptr(proofs), stride, _ptr(offsets),
                                               C.c_void_p(stream or 0)), 'zka_proofs_unpack')

    # ------------------------------------------------------------------ layer-wise ops
    def tom_commit_batch(self, params, v: np.ndarray, r: np.ndarray) -> np.ndarray:
        count = v.shape[0]
        out = np.zeros((count, self.wp), np.uint8)
        self._check(self.lib.zka_tom_commit_batch(self.ctx, params, count, _ptr(v), _ptr(r), _ptr(out)),
                    'zka_tom_commit_batch')
        return out

    def p256_mul_batch(self, base: Optional[np.ndarray], k: np.ndarray) -> np.ndarray:
        count = k.shape[0]
        out = np.zeros((count, 65), np.uint8)
        self._check(self.lib.zka_p256_mul_batch(self.ctx, count, _ptr(base), _ptr(k), _ptr(out)), 'zka_p256_mul_batch')
        return out

    def field_op_batch(self, field: int, op: int, a: np.ndarray, b: Optional[np.ndarray]) -> np.ndarray:
        count, nb = a.shape
        out = np.zeros((count, nb), np.uint8)
        self._check(self.lib.zka_field_op_batch(self.ctx, field, op, count, _ptr(a), _ptr(b), _ptr(out)),
                    'zka_field_op_batch')
        return out

    def hash80_batch(self, msgs: np.ndarray, lens: np.ndarray) -> np.ndarray:
        count, stride = msgs.shape
        out = np.zeros((count, 10), np.uint8)
        self._check(self.lib.zka_hash80_batch(self.ctx, count, _ptr(msgs), stride, _ptr(lens), _ptr(out)),
                    'zka_hash80_batch')
        return out
