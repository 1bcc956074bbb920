"""Seeded mode against hedged mode (each proof's seed derived on the GPU from the caller's seed, the statement and the
signature: include/zkattest.h, "Hedged seeds"), in one process.

Workloads (SecLevel 80): config2 (8192 proofs, ring 256), config1 (1024 proofs, ring 8) and a ring set (8192 rows over
64 rings of 8 ... 1024 entries).  For each: warm-up, then three rounds that alternate the modes, each call timed with a
device synchronise at its end:
  * seeded   zka_prove_batch_seeded with random seeds;
  * hedged   zka_prove_batch_hedged with random seeds;
  * hedged0  zka_prove_batch_hedged with seeds = NULL (deterministic);
device-resident (inputs, seeds and outputs in HBM) and host-buffer end to end.  Then a checksum showing the hedged proofs
equal the seeded proofs on the seeds zka_hedge_seeds derives, and one profiled pass for the time of SeedHedgeTask and
RingDigestTask.  Last, one ring of 2^20 entries: RingDigestTask (1024 leaves, then the root) timed on its own.

    python tools/hedged_bench.py [--out FILE.json] [--workloads config2,config1,rings,digest]

Each run prints one JSON line; --out also writes the whole record to FILE.json.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from zkp_ecdsa_b200 import synth  # noqa: E402
from zkp_ecdsa_b200 import api  # noqa: E402

SEC = 80
WORKLOADS = {'config1': (1024, 8), 'config2': (8192, 256)}
MODES = ('seeded', 'hedged', 'hedged0')
RING_SET_SIZES = [8 << (i % 8) for i in range(64)]    # 8, 16, ..., 1024, eight times


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return t.data_ptr()


def run(eng, wname):
    L = eng.lib
    params = eng.generate_params_list(SEC, rnd=synth.params_rnd(0))
    P = params.handle
    if wname == 'rings':
        B = 8192
        ring_of = np.random.Generator(np.random.PCG64(1)).integers(0, len(RING_SET_SIZES), B).astype(np.uint32)
        wl = synth.RingsWorkload(B, RING_SET_SIZES, ring_of, seed=0)
        rings = eng.load_rings(wl.rings)
        ps = L.proof_max_len(max(RING_SET_SIZES), SEC)
        d_ring_of = dev(ring_of.view(np.int32))
    else:
        B, N = WORKLOADS[wname]
        wl = synth.Workload(B, N, seed=0, distinct_signers=min(B, N))
        ps = L.proof_max_len(N, SEC)
        d_ring = dev(wl.ring)
    seeds = np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32).copy()
    d_msg, d_sig, d_pk, d_which, d_seed = dev(wl.msg_hash), dev(wl.sig), dev(wl.pk), dev(wl.which.view(np.int32)), dev(seeds)
    d_pr = {m: torch.zeros(B * ps, dtype=torch.uint8, device='cuda') for m in MODES + ('check',)}
    d_len = {m: torch.zeros(B, dtype=torch.int32, device='cuda') for m in MODES + ('check',)}
    d_st = torch.zeros(B, dtype=torch.int32, device='cuda')
    d_derived = torch.zeros(B * 32, dtype=torch.uint8, device='cuda')

    def call(m, msg, sig, pk, which, sd, pr, ln, st):
        fn = 'seeded' if m in ('seeded', 'check') else 'hedged'
        if wname == 'rings':
            rof = ptr(d_ring_of) if isinstance(msg, int) else ring_of
            getattr(L, f'prove_batch_rings_{fn}')(P, rings.handle, rof, B, msg, sig, pk, which, sd, pr, ps, ln, st)
        else:
            ring = ptr(d_ring) if isinstance(msg, int) else wl.ring
            getattr(L, f'prove_batch_{fn}')(P, B, msg, sig, pk, which, ring, N, sd, pr, ps, ln, st)

    def prove_dev(m, sd=None):
        sd = sd if sd is not None else (None if m == 'hedged0' else ptr(d_seed))
        call(m, ptr(d_msg), ptr(d_sig), ptr(d_pk), ptr(d_which), sd, ptr(d_pr[m]), ptr(d_len[m]), ptr(d_st))

    h_pr = np.zeros((B, ps), np.uint8)
    h_len = np.zeros(B, np.uint32)
    h_st = np.zeros(B, np.int32)

    def e2e(m):
        s = None if m == 'hedged0' else np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32)
        call(m, wl.msg_hash, wl.sig, wl.pk, wl.which, s, h_pr, h_len, h_st)

    for m in MODES:                                    # warm-up of every shape
        prove_dev(m)
        e2e(m)
    res = {'prove_dev': {m: [] for m in MODES}, 'prove_e2e': {m: [] for m in MODES}}
    for _ in range(3):
        for m in MODES:
            res['prove_dev'][m].append(B / timed(lambda: prove_dev(m)))
            res['prove_e2e'][m].append(B / timed(lambda: e2e(m)))
            assert not d_st.cpu().numpy().any() and not h_st.any()
    # equality at the timed size: hedged proofs against seeded proofs on the derived seeds
    if wname == 'rings':
        L.hedge_seeds_rings(P, rings.handle, ptr(d_ring_of), B, ptr(d_msg), ptr(d_sig), ptr(d_pk), ptr(d_which), ptr(d_seed),
                            ptr(d_derived))
    else:
        L.hedge_seeds(P, B, ptr(d_msg), ptr(d_sig), ptr(d_pk), ptr(d_which), ptr(d_ring), N, ptr(d_seed), ptr(d_derived))
    prove_dev('hedged')
    prove_dev('check', ptr(d_derived))
    torch.cuda.synchronize()
    sums = {m: hashlib.sha256(d_pr[m].cpu().numpy().tobytes() + d_len[m].cpu().numpy().tobytes()).hexdigest()
            for m in ('hedged', 'check')}
    assert sums['hedged'] == sums['check'], sums
    # kernel time of the derivation, in a profiled pass of its own
    L.set_profiling(True)
    L.profile_reset()
    prove_dev('hedged')
    torch.cuda.synchronize()
    prof = L.profile()
    L.set_profiling(False)
    kern = {k.split('::')[-1]: v for k, v in prof.items() if 'Hedge' in k or 'Digest' in k or 'SeedProve' in k}
    total_ms = sum(v['ms'] for v in prof.values())
    if wname == 'rings':
        rings.close()
    params.close()
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    return {'workload': wname, 'B': B, 'N': RING_SET_SIZES if wname == 'rings' else N, 'sec_level': SEC,
            'rates_per_s': res,
            'median_per_s': {k: {m: med(v) for m, v in d.items()} for k, d in res.items()},
            'hedged_over_seeded_median': {k: med(d['hedged']) / med(d['seeded']) for k, d in res.items()},
            'kernels_profiled': kern, 'profiled_kernel_ms_total': total_ms,
            'checksum_hedged_equals_seeded_on_derived': sums['hedged']}


def run_digest(eng, reps=5):
    """RingDigestTask on one ring of 2^20 entries: zka_hedge_seeds of one row, profiled, and the call timed."""
    L = eng.lib
    params = eng.generate_params_list(SEC, rnd=synth.params_rnd(0))
    N = 1 << 20
    ring = np.frombuffer(synth.Drbg(0, 'digest-ring').bytes(32 * N), np.uint8).reshape(N, 32).copy()
    wl = synth.Workload(1, 8, seed=0)
    d_ring = dev(ring)
    out = np.zeros((1, 32), np.uint8)

    def once():
        L.hedge_seeds(params.handle, 1, wl.msg_hash, wl.sig, wl.pk, wl.which, ptr(d_ring), N, None, out)
    once()
    call_ms = [1e3 * timed(once) for _ in range(reps)]
    L.set_profiling(True)
    L.profile_reset()
    for _ in range(reps):
        once()
    torch.cuda.synchronize()
    prof = L.profile()
    L.set_profiling(False)
    params.close()
    kern = {k.split('::')[-1]: v for k, v in prof.items()}
    return {'workload': 'digest', 'N': N, 'leaves': N // 1024, 'calls': reps, 'call_ms': call_ms, 'kernels_profiled': kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='write the whole record here as JSON')
    ap.add_argument('--workloads', default='config2,config1,rings,digest')
    a = ap.parse_args()
    eng = api.Engine(0)
    out = {'card': card(), 'lanes': eng.lib.config()['lanes'], 'runs': []}
    for w in a.workloads.split(','):
        r = run_digest(eng) if w == 'digest' else run(eng, w)
        out['runs'].append(r)
        print(json.dumps(r), flush=True)
    out['card_after'] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps({'card': out['card']}))


if __name__ == '__main__':
    main()
