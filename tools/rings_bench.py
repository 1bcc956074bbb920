"""Ring sets against the routes a caller has without them, in one process (SecLevel 80, 20 samples, seeded randomness).

  (a) own8:         8192 rows, every signer with a ring of 8 of its own (8192 rings in one set)
  (b) mixed64:      8192 rows over 64 rings of 8 .. 1024 entries (depths 3 .. 10), rows grouped by depth;
      mixed64_interleaved: the first 512 rows of the same set with the depth changing from row to row (a pass per row)
  (c) per_ring_256: the first 256 rows of (a) as 256 one-ring calls (zka_prove_batch_seeded / zka_verify_batch_seeded);
      config1:      bench.py's config1, 1024 proofs sharing one ring of 8, as the one-ring reference

For each: warm-up, then three timed rounds (device synchronise at the end of each) of device-resident prove and verify
(inputs, seeds and outputs in HBM) and of end-to-end prove and verify with host buffers; the interleaved and per-ring
cases are timed once per round on the device only.  Proof bytes of (a) and (c) on their common rows are compared.

    python tools/rings_bench.py [--out FILE.json]

Each case prints one JSON line; --out also writes the whole record to FILE.json.
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

from zkp_ecdsa_b200 import synth  # noqa: E402
from zkp_ecdsa_b200.capi import ZkaLib  # noqa: E402

SEC = 80
K = 20
B = 8192


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


def seeds(rows, tag):
    return np.frombuffer(synth.Drbg(rows, f'rings-bench-{tag}').bytes(32 * rows), np.uint8).reshape(rows, 32).copy()


class Case:
    """The device and host buffers of one ring-set workload and its prove / verify calls."""

    def __init__(self, L: ZkaLib, P, wl, rows=None):
        self.L, self.P = L, P
        idx = np.arange(wl.B) if rows is None else np.asarray(rows)
        self.B = len(idx)
        self.ring_of = wl.ring_of[idx].copy()
        self.msg, self.sig, self.pk, self.which = (getattr(wl, k)[idx].copy() for k in ('msg_hash', 'sig', 'pk', 'which'))
        self.ps = L.proof_max_len(max(wl.sizes[int(r)] for r in np.unique(self.ring_of)), SEC)
        self.seeds, self.vseeds = seeds(self.B, 'p'), seeds(self.B, 'v')
        self.rs = L.rings_create(np.array(wl.sizes, np.uint32), wl.keys)
        self.d = {k: dev(v) for k, v in (('ro', self.ring_of.view(np.int32)), ('msg', self.msg), ('sig', self.sig), ('pk', self.pk),
                                         ('which', self.which.view(np.int32)), ('seed', self.seeds), ('vseed', self.vseeds))}
        self.d['pr'] = torch.zeros(self.B * self.ps, dtype=torch.uint8, device='cuda')
        self.d['len'] = torch.zeros(self.B, dtype=torch.int32, device='cuda')
        self.d['st'] = torch.zeros(self.B, dtype=torch.int32, device='cuda')
        self.d['ok'] = torch.zeros(self.B, dtype=torch.uint8, device='cuda')
        self.h_pr = np.zeros((self.B, self.ps), np.uint8)
        self.h_len, self.h_st, self.h_ok = np.zeros(self.B, np.uint32), np.zeros(self.B, np.int32), np.zeros(self.B, np.uint8)

    def p(self, k):
        return self.d[k].data_ptr()

    def prove_dev(self):
        self.L.prove_batch_rings_seeded(self.P, self.rs, self.p('ro'), self.B, self.p('msg'), self.p('sig'), self.p('pk'), self.p('which'),
                                        self.p('seed'), self.p('pr'), self.ps, self.p('len'), self.p('st'))

    def verify_dev(self):
        self.L.verify_batch_rings_seeded(self.P, self.rs, self.p('ro'), self.B, self.p('msg'), self.p('pr'), self.ps, self.p('len'),
                                         self.p('vseed'), K, self.p('ok'), self.p('st'))

    def prove_e2e(self):
        self.L.prove_batch_rings_seeded(self.P, self.rs, self.ring_of, self.B, self.msg, self.sig, self.pk, self.which, self.seeds,
                                        self.h_pr, self.ps, self.h_len, self.h_st)

    def verify_e2e(self):
        self.L.verify_batch_rings_seeded(self.P, self.rs, self.ring_of, self.B, self.msg, self.h_pr, self.ps, self.h_len, self.vseeds,
                                         K, self.h_ok, self.h_st)

    def check(self):
        torch.cuda.synchronize()
        assert not self.d['st'].cpu().numpy().any() and self.d['ok'].cpu().numpy().all()

    def proofs(self):
        torch.cuda.synchronize()
        return self.d['pr'].cpu().numpy().reshape(self.B, self.ps), self.d['len'].cpu().numpy().view(np.uint32)

    def close(self):
        self.L.rings_destroy(self.rs)


def rates(case, kinds, rounds=3):
    fns = {'prove_dev': case.prove_dev, 'verify_dev': case.verify_dev, 'prove_e2e': case.prove_e2e, 'verify_e2e': case.verify_e2e}
    for k in kinds:                                      # warm-up of every shape
        fns[k]()
    out = {k: [] for k in kinds}
    for _ in range(rounds):
        for k in kinds:
            out[k].append(case.B / timed(fns[k]))
        case.check()
    if 'verify_e2e' in kinds:
        assert not case.h_st.any() and case.h_ok.all()
    return out


def summary(name, case, depth, res, extra=None):
    """depth[r]: the depth of ring r; a call makes one pass per run of rows of equal depth."""
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    r = {'case': name, 'rows': case.B, 'rings_used': int(len(np.unique(case.ring_of))),
         'passes': int(1 + np.count_nonzero(np.diff([depth[int(r)] for r in case.ring_of]))),
         'rates_per_s': res, 'median_per_s': {k: med(v) for k, v in res.items()}}
    for k in ('prove_dev', 'verify_dev', 'prove_e2e', 'verify_e2e'):
        if k not in res:
            r['median_per_s'][k] = 'not measured'
    r.update(extra or {})
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='write the whole record here as JSON')
    a = ap.parse_args()
    L = ZkaLib(device=0)
    hn, hp = L.params_generate(synth.params_rnd(0))
    P = L.params_create(hn, hp, SEC)
    out = {'card': card(), 'lanes': L.config()['lanes'], 'sec_level': SEC, 'samples': K, 'randomness': 'seeded', 'cases': []}

    def emit(r):
        out['cases'].append(r)
        print(json.dumps(r), flush=True)

    # (a) every signer with a ring of 8 of its own
    wa = synth.RingsWorkload(B, [8] * B, np.arange(B), seed=1)
    ca = Case(L, P, wa)
    emit(summary('own8', ca, [3] * B, rates(ca, ('prove_dev', 'verify_dev', 'prove_e2e', 'verify_e2e'))))
    pa, la = ca.proofs()
    # (c) the only route without ring sets: the first 256 rows of (a), one one-ring call each, on the same seeds
    n1 = 256
    d_keys = dev(wa.keys)
    ps1 = L.proof_max_len(8, SEC)
    d_pr1 = torch.zeros(n1 * ps1, dtype=torch.uint8, device='cuda')
    d_len1 = torch.zeros(n1, dtype=torch.int32, device='cuda')
    d_ok1 = torch.zeros(n1, dtype=torch.uint8, device='cuda')

    def per_ring_prove():
        for i in range(n1):
            L.prove_batch_seeded(P, 1, ca.p('msg') + 32 * i, ca.p('sig') + 64 * i, ca.p('pk') + 65 * i, ca.p('which') + 4 * i,
                                 d_keys.data_ptr() + 32 * 8 * i, 8, ca.p('seed') + 32 * i, d_pr1.data_ptr() + ps1 * i, ps1,
                                 d_len1.data_ptr() + 4 * i, ca.p('st') + 4 * i)

    def per_ring_verify():
        for i in range(n1):
            L.verify_batch_seeded(P, 1, ca.p('msg') + 32 * i, d_keys.data_ptr() + 32 * 8 * i, 8, d_pr1.data_ptr() + ps1 * i, ps1,
                                  d_len1.data_ptr() + 4 * i, ca.p('vseed') + 32 * i, K, d_ok1.data_ptr() + i, ca.p('st') + 4 * i)
    per_ring_prove()
    per_ring_verify()
    pr_rates = {'prove_dev': [], 'verify_dev': []}
    for _ in range(3):
        pr_rates['prove_dev'].append(n1 / timed(per_ring_prove))
        pr_rates['verify_dev'].append(n1 / timed(per_ring_verify))
    torch.cuda.synchronize()
    assert d_ok1.cpu().numpy().all() and not ca.d['st'].cpu().numpy()[:n1].any()
    p1 = d_pr1.cpu().numpy().reshape(n1, ps1)
    l1 = d_len1.cpu().numpy().view(np.uint32)
    same = bool(np.array_equal(l1, la[:n1]) and all(p1[i, :l1[i]].tobytes() == pa[i, :la[i]].tobytes() for i in range(n1)))
    assert same
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    emit({'case': 'per_ring_256', 'rows': n1, 'calls': n1, 'rates_per_s': pr_rates,
          'median_per_s': {'prove_dev': med(pr_rates['prove_dev']), 'verify_dev': med(pr_rates['verify_dev']),
                           'prove_e2e': 'not measured', 'verify_e2e': 'not measured'},
          'proofs_equal_own8_rows': same})
    ca.close()
    # config1: one shared ring of 8 (bench.py's workload), one-ring calls
    w1 = synth.Workload(1024, 8, seed=0, distinct_signers=8)
    c1 = {k: dev(v) for k, v in (('msg', w1.msg_hash), ('sig', w1.sig), ('pk', w1.pk), ('which', w1.which.view(np.int32)),
                                 ('ring', w1.ring), ('seed', seeds(1024, 'c1p')), ('vseed', seeds(1024, 'c1v')))}
    c1['pr'] = torch.zeros(1024 * ps1, dtype=torch.uint8, device='cuda')
    c1['len'] = torch.zeros(1024, dtype=torch.int32, device='cuda')
    c1['st'] = torch.zeros(1024, dtype=torch.int32, device='cuda')
    c1['ok'] = torch.zeros(1024, dtype=torch.uint8, device='cuda')
    q = lambda k: c1[k].data_ptr()   # noqa: E731
    fns = {'prove_dev': lambda: L.prove_batch_seeded(P, 1024, q('msg'), q('sig'), q('pk'), q('which'), q('ring'), 8, q('seed'), q('pr'),
                                                     ps1, q('len'), q('st')),
           'verify_dev': lambda: L.verify_batch_seeded(P, 1024, q('msg'), q('ring'), 8, q('pr'), ps1, q('len'), q('vseed'), K, q('ok'),
                                                       q('st'))}
    for f in fns.values():
        f()
    c1r = {k: [] for k in fns}
    for _ in range(3):
        for k, f in fns.items():
            c1r[k].append(1024 / timed(f))
    torch.cuda.synchronize()
    assert c1['ok'].cpu().numpy().all() and not c1['st'].cpu().numpy().any()
    emit({'case': 'config1', 'rows': 1024, 'rates_per_s': c1r,
          'median_per_s': {k: med(v) for k, v in c1r.items()} | {'prove_e2e': 'not measured', 'verify_e2e': 'not measured'}})
    del c1
    # (b) 64 rings of 8 .. 1024 entries, rows grouped by depth, then interleaved
    sizes = [8 << (i % 8) for i in range(64)]
    depth = [(s - 1).bit_length() for s in sizes]
    ring_of = np.array(sorted((b % 64 for b in range(B)), key=lambda r: (depth[r], r)), np.uint32)
    wb = synth.RingsWorkload(B, sizes, ring_of, seed=2)
    cb = Case(L, P, wb)
    emit(summary('mixed64', cb, depth, rates(cb, ('prove_dev', 'verify_dev', 'prove_e2e', 'verify_e2e'))))
    cb.close()
    # the same set with the depth changing from row to row: rows r0 of ring 0, then ring 1, ... (one pass per row)
    n_il = 512
    first = {r: np.flatnonzero(ring_of == r) for r in range(64)}
    il = [int(first[b % 64][b // 64]) for b in range(n_il)]
    ci = Case(L, P, wb, il)
    emit(summary('mixed64_interleaved', ci, depth, rates(ci, ('prove_dev', 'verify_dev')),
                 {'rows_of': 'the first 512 rows, round-robin over the 64 rings'}))
    ci.close()
    L.params_destroy(P)
    out['card_after'] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps({'card': out['card']}))


if __name__ == '__main__':
    main()
