"""Prove rate with the self-check off and on (include/zkattest.h, "Self-checked proving"), in one process.

Workload: config2 (8192 proofs, ring 256, SecLevel 80).  Cases: device-resident buffers (inputs, randomness and outputs in
HBM) and host buffers end to end, each with hedged seeds (zka_prove_batch_hedged, random caller seeds) and with a tape
(zka_prove_batch).  For each case: one warm-up call per mode, then three rounds that alternate off and on, each call timed
with a device synchronise at its end.  Then a checksum that the checked proofs equal the unchecked ones, the self-check
counters, and the device memory in use after each mode's warm-up (the library's workspace pools only grow, so this is
the running peak of the process; cudaMemGetInfo, and the process's own line of nvidia-smi when it has one).

    python tools/self_check_bench.py [--out FILE.json] [--cases dev-hedged,dev-tape,host-hedged,host-tape]

Each case prints one JSON line; --out also writes the whole record to FILE.json.
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

SEC, B, N = 80, 8192, 256
MODES = ('off', 'on')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def mem_gb():
    """device memory in use (all processes, cudaMemGetInfo) and this process's own (nvidia-smi), in GB"""
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    own = None
    q = subprocess.run(['nvidia-smi', '--query-compute-apps=pid,used_memory', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True)
    if q.returncode == 0:
        for line in q.stdout.strip().splitlines():
            pid, used = (s.strip() for s in line.split(','))
            if pid == str(os.getpid()):
                own = float(used) / 1024
    return {'device_used_gb': (total - free) / 2**30, 'process_used_gb': own}


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(eng, params, case):
    L = eng.lib
    P = params.handle
    where, kind = case.split('-')
    wl = synth.Workload(B, N, seed=0, distinct_signers=N)
    ps = L.proof_max_len(N, SEC)
    ts = L.prove_tape_len(N, SEC)
    tape = synth.random_tape(B, ts, seed=1) if kind == 'tape' else None
    if where == 'dev':
        d = {k: dev(v) for k, v in (('msg', wl.msg_hash), ('sig', wl.sig), ('pk', wl.pk), ('which', wl.which.view(np.int32)),
                                     ('ring', wl.ring))}
        if tape is not None:
            d['tape'] = dev(tape)
        out = {m: (torch.zeros(B * ps, dtype=torch.uint8, device='cuda'), torch.zeros(B, dtype=torch.int32, device='cuda'),
                   torch.zeros(B, dtype=torch.int32, device='cuda')) for m in MODES}
        args = [d['msg'].data_ptr(), d['sig'].data_ptr(), d['pk'].data_ptr(), d['which'].data_ptr(), d['ring'].data_ptr()]
        outs = {m: (o[0].data_ptr(), ps, o[1].data_ptr(), o[2].data_ptr()) for m, o in out.items()}
        tape_arg = d['tape'].data_ptr() if tape is not None else None
    else:
        out = {m: (np.zeros((B, ps), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)) for m in MODES}
        args = [wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring]
        outs = {m: (o[0], ps, o[1], o[2]) for m, o in out.items()}
        tape_arg = tape
    seeds = np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32).copy()
    d_seeds = dev(seeds) if where == 'dev' else None

    def prove(m):
        L.set_option('self_check', 2 if m == 'on' else 1)
        if kind == 'tape':
            L.prove_batch(P, B, *args[:4], args[4], N, tape_arg, ts, *outs[m])
        else:
            L.prove_batch_hedged(P, B, *args[:4], args[4], N, d_seeds.data_ptr() if d_seeds is not None else seeds, *outs[m])

    mem = {'before': mem_gb()}
    for m in MODES:                                    # warm-up of every shape
        prove(m)
        mem[f'after_{m}_warmup'] = mem_gb()
    r0 = (L.stat('self_check_rows'), L.stat('self_check_fail'))
    rates = {m: [] for m in MODES}
    for _ in range(3):
        for m in MODES:
            rates[m].append(B / timed(lambda: prove(m)))
    L.set_option('self_check', 1)
    counts = (L.stat('self_check_rows') - r0[0], L.stat('self_check_fail') - r0[1])

    def host(o):
        pr, ln, st = (x.cpu().numpy() if torch.is_tensor(x) else x for x in o)
        return pr.reshape(B, ps), ln.view(np.uint32), st
    res = {m: host(out[m]) for m in MODES}
    for m in MODES:
        assert not res[m][2].any(), (m, np.unique(res[m][2]))
    # each proof up to its length (with host buffers the bytes of a row beyond it are whatever the staging buffer held)
    sums = {m: hashlib.sha256(b''.join(res[m][0][b, :n].tobytes() for b, n in enumerate(res[m][1])) + res[m][1].tobytes()
                              + res[m][2].tobytes()).hexdigest() for m in MODES}
    assert sums['off'] == sums['on'], sums
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    return {'case': case, 'B': B, 'N': N, 'sec_level': SEC, 'chunk': L.config()['chunk'], 'rates_per_s': rates,
            'median_per_s': {m: med(v) for m, v in rates.items()}, 'on_over_off_median': med(rates['on']) / med(rates['off']),
            'self_check_rows': counts[0], 'self_check_fail': counts[1], 'memory': mem,
            'checksum_on_equals_off': sums['on']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='write the whole record here as JSON')
    ap.add_argument('--cases', default='dev-hedged,dev-tape,host-hedged,host-tape')
    a = ap.parse_args()
    eng = api.Engine(0)
    params = eng.generate_params_list(SEC, rnd=synth.params_rnd(0))
    out = {'card': card(), 'lanes': eng.lib.config()['lanes'], 'runs': []}
    for c in a.cases.split(','):
        r = run(eng, params, c)
        out['runs'].append(r)
        print(json.dumps(r), flush=True)
    params.close()
    out['card_after'] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps({'card': out['card']}))


if __name__ == '__main__':
    main()
