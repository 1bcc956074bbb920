"""Cost of traceable proofs (include/zkattest.h, "Traceable proofs") against the untraced calls, in one process.

Workload: config2 (8192 proofs, ring 256, SecLevel 80, tape randomness).  Cases: prove and verify (20 samples), each with
device-resident buffers and with host buffers end to end; one warm-up call per mode, then three rounds that alternate
untraced and traced, each call timed with a device synchronise at its end.  Then zka_open_batch over the 8192 traced
proofs against the ring of 256 and against a ring of 2^20 entries holding the same keys, each timed three times after a
warm-up.  Rows are checked: every traced proof verifies, its base bytes are the untraced proof, and every row opens to
its `which`.

    python tools/traced_bench.py [--out FILE.json]

Each case prints one JSON line; --out also writes the whole record (with the card's name and power limit) to FILE.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from zkp_ecdsa_b200 import api, synth  # noqa: E402
from zkp_ecdsa_b200 import verify_tape as VT  # noqa: E402

SEC, B, N, K = 80, 8192, 256, 20
MODES = ('untraced', 'traced')
SK = 0x5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed5eed


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


def med(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    eng = api.Engine(0)
    L = eng.lib
    params = eng.generate_params_list(SEC, rnd=synth.params_rnd(0))
    P = params.handle
    _, Y = eng.trace_keypair(SK)
    T = L.trace_len()
    wl = synth.Workload(B, N, seed=0, distinct_signers=N)
    ts = L.prove_tape_len(N, SEC) + 128
    ps = L.proof_max_len(N, SEC) + T
    tape = synth.random_tape(B, ts, seed=1)
    vts = L.verify_tape_len_ex(N, SEC, K)
    vtape = VT.random_verify_tape(B, vts, N, SEC, seed=2)
    out = {'card': card(), 'lanes': L.config()['lanes'], 'B': B, 'N': N, 'sec_level': SEC, 'samples': K, 'runs': []}
    host = {'msg': wl.msg_hash, 'sig': wl.sig, 'pk': wl.pk, 'which': wl.which, 'ring': wl.ring, 'tape': tape, 'vtape': vtape}
    rows = {}
    for where in ('dev', 'host'):
        if where == 'dev':
            d = {k: dev(v.view(np.int32) if k == 'which' else v) for k, v in host.items()}
            ptr = {k: v.data_ptr() for k, v in d.items()}
            bufs = {m: (torch.zeros(B * ps, dtype=torch.uint8, device='cuda'), torch.zeros(B, dtype=torch.int32, device='cuda'),
                        torch.zeros(B, dtype=torch.int32, device='cuda')) for m in MODES}
            o = {m: tuple(x.data_ptr() for x in b) for m, b in bufs.items()}
            vo = (torch.zeros(B, dtype=torch.uint8, device='cuda'), torch.zeros(B, dtype=torch.int32, device='cuda'))
            vout = tuple(x.data_ptr() for x in vo)
        else:
            ptr = host
            bufs = {m: (np.zeros((B, ps), np.uint8), np.zeros(B, np.uint32), np.zeros(B, np.int32)) for m in MODES}
            o = bufs
            vo = (np.zeros(B, np.uint8), np.zeros(B, np.int32))
            vout = vo

        def prove(m):
            pr, ln, st = o[m]
            if m == 'traced':
                L.prove_batch_traced(P, B, ptr['msg'], ptr['sig'], ptr['pk'], ptr['which'], ptr['ring'], N, ptr['tape'], ts, pr, ps, ln, st, Y)
            else:
                L.prove_batch(P, B, ptr['msg'], ptr['sig'], ptr['pk'], ptr['which'], ptr['ring'], N, ptr['tape'], ts, pr, ps, ln, st)

        def verify(m):
            pr, ln, _ = o[m]
            if m == 'traced':
                L.verify_batch_traced(P, B, ptr['msg'], ptr['ring'], N, pr, ps, ln, ptr['vtape'], vts, vout[0], vout[1], K, Y)
            else:
                L.verify_batch_ex(P, B, ptr['msg'], ptr['ring'], N, pr, ps, ln, ptr['vtape'], vts, vout[0], vout[1], K)

        for stage, fn in (('prove', prove), ('verify', verify)):
            for m in MODES:
                fn(m)
            if stage == 'verify':
                okv = vo[0].cpu().numpy() if torch.is_tensor(vo[0]) else vo[0]
                assert okv.all()
            rates = {m: [] for m in MODES}
            for _ in range(3):
                for m in MODES:
                    rates[m].append(B / timed(lambda: fn(m)))
            r = {'case': f'{where}-{stage}', 'rates_per_s': rates, 'median_per_s': {m: med(v) for m, v in rates.items()},
                 'traced_over_untraced_median': med(rates['traced']) / med(rates['untraced'])}
            out['runs'].append(r)
            print(json.dumps(r), flush=True)
        got = {m: tuple(x.cpu().numpy() if torch.is_tensor(x) else x for x in bufs[m]) for m in MODES}
        pu, lu, su = got['untraced']
        pt, lt, st = got['traced']
        pu, pt, lu, lt = pu.reshape(B, ps), pt.reshape(B, ps), lu.view(np.uint32), lt.view(np.uint32)
        assert not su.any() and not st.any() and (lt == lu + T).all()
        assert all(pt[b, :lu[b]].tobytes() == pu[b, :lu[b]].tobytes() for b in range(B))
        rows[where] = (pt, lt)
    # the opener on the host-buffer rows, against the ring and against 2^20 entries holding the same keys
    pt, lt = rows['host']
    big = np.random.default_rng(3).integers(0, 256, size=(1 << 20, 32), dtype=np.uint8)
    slots = np.random.default_rng(4).permutation(1 << 20)[:N]
    big[slots] = wl.ring
    for name, ring, expect in (('open-ring256', wl.ring, wl.which), ('open-ring2^20', big, slots[wl.which])):
        fn = lambda: eng.open_batch(params, SK, wl.msg_hash, ring, pt, lt)   # noqa: E731
        idx, ost = fn()
        assert not ost.any() and (idx == expect).all()
        times = [timed(fn) for _ in range(3)]
        r = {'case': name, 'ring': int(ring.shape[0]), 'seconds': times, 'median_rows_per_s': B / med(times)}
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
