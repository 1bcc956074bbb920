"""Ring-set rows in arrival order against the same rows grouped by ring depth, in one process (SecLevel 80, 20 samples).

  mixed64_grouped / mixed64_interleaved: 8192 rows over the 64 rings of 8 .. 1024 entries of tools/rings_bench.py case b
      (depths 3 .. 10), the SAME rows grouped by depth and with the depth changing on every row
  own8:    8192 rows, every signer with a ring of 8 of its own (tools/rings_bench.py case a)
  config1: bench.py's config1, 1024 proofs sharing one ring of 8, through the one-ring calls

Warm-up of every shape, then three rounds that alternate the cases; every timing ends in a device synchronise.  Prove and
verify are device-resident (inputs, randomness and outputs in HBM), with seeded randomness and, for the two mixed64
cases, with tapes as well.  Proof checksums of the interleaved and grouped runs are compared row by row.  A profiled
pass of its own (per-kernel CUDA events, one lane) then gives GkPolyTask, VGkSumTask and VGkTask of both orders and
their share of all kernel time.

    python tools/rings_mixed_bench.py [--out FILE.json]
"""
import argparse
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rings_bench import B, K, SEC, Case, card, dev, seeds, timed  # noqa: E402
from zkp_ecdsa_b200 import synth  # noqa: E402
from zkp_ecdsa_b200 import verify_tape as VT  # noqa: E402
from zkp_ecdsa_b200.capi import ZkaLib  # noqa: E402

GK_TASKS = ('GkPolyTask', 'VGkSumTask', 'VGkTask')


class TapeCase(Case):
    """A Case that also holds, on the device, the tapes its seeds stand for (each row laid out for its own ring)."""

    def __init__(self, L, P, wl, rows=None):
        super().__init__(L, P, wl, rows)
        if rows is not None:   # a row keeps the seeds it has in the whole workload, so the two orders give the same proofs
            self.seeds, self.vseeds = seeds(wl.B, 'p')[np.asarray(rows)].copy(), seeds(wl.B, 'v')[np.asarray(rows)].copy()
            self.d['seed'], self.d['vseed'] = dev(self.seeds), dev(self.vseeds)
        nmax = max(wl.sizes[int(r)] for r in np.unique(self.ring_of))
        self.ts, self.vts = L.prove_tape_len(nmax, SEC), L.verify_tape_len_ex(nmax, SEC, K)
        tape, vtape = np.zeros((self.B, self.ts), np.uint8), np.zeros((self.B, self.vts), np.uint8)
        for r in np.unique(self.ring_of):
            rows_r = np.flatnonzero(self.ring_of == r)
            t = L.seed_tape(0, self.seeds[rows_r].copy(), wl.sizes[int(r)], SEC, K)
            tape[rows_r, :t.shape[1]] = t
            t = L.seed_tape(1, self.vseeds[rows_r].copy(), wl.sizes[int(r)], SEC, K)
            vtape[rows_r, :t.shape[1]] = t
        self.d['tape'], self.d['vtape'] = dev(tape), dev(vtape)

    def prove_tape(self):
        self.L.prove_batch_rings(self.P, self.rs, self.p('ro'), self.B, self.p('msg'), self.p('sig'), self.p('pk'), self.p('which'),
                                 self.p('tape'), self.ts, self.p('pr'), self.ps, self.p('len'), self.p('st'))

    def verify_tape(self):
        self.L.verify_batch_rings(self.P, self.rs, self.p('ro'), self.B, self.p('msg'), self.p('pr'), self.ps, self.p('len'),
                                  self.p('vtape'), self.vts, K, self.p('ok'), self.p('st'))

    def checksums(self):
        pr, ln = self.proofs()
        return [hashlib.sha256(pr[b, :ln[b]].tobytes()).hexdigest() for b in range(self.B)]


def config1(L, P):
    w1 = synth.Workload(1024, 8, seed=0, distinct_signers=8)
    ps1 = L.proof_max_len(8, SEC)
    c1 = {k: dev(v) for k, v in (('msg', w1.msg_hash), ('sig', w1.sig), ('pk', w1.pk), ('which', w1.which.view(np.int32)),
                                 ('ring', w1.ring), ('seed', seeds(1024, 'c1p')), ('vseed', seeds(1024, 'c1v')))}
    c1['pr'] = torch.zeros(1024 * ps1, dtype=torch.uint8, device='cuda')
    for k, t in (('len', torch.int32), ('st', torch.int32), ('ok', torch.uint8)):
        c1[k] = torch.zeros(1024, dtype=t, device='cuda')
    q = lambda k: c1[k].data_ptr()   # noqa: E731

    def check():
        torch.cuda.synchronize()
        assert c1['ok'].cpu().numpy().all() and not c1['st'].cpu().numpy().any()
    return {'rows': 1024, 'check': check, 'keep': c1,
            'prove_dev': lambda: L.prove_batch_seeded(P, 1024, q('msg'), q('sig'), q('pk'), q('which'), q('ring'), 8, q('seed'), q('pr'),
                                                      ps1, q('len'), q('st')),
            'verify_dev': lambda: L.verify_batch_seeded(P, 1024, q('msg'), q('ring'), 8, q('pr'), ps1, q('len'), q('vseed'), K, q('ok'),
                                                        q('st'))}


def of_case(c, tape):
    r = {'rows': c.B, 'check': c.check, 'prove_dev': c.prove_dev, 'verify_dev': c.verify_dev}
    if tape:
        r.update(prove_tape=c.prove_tape, verify_tape=c.verify_tape)
    return r


def gk_profile(L, case):
    """One profiled prove + verify of `case` on one lane: ms of the GK polynomial kernels and of all kernels."""
    lanes = L.config()['lanes']
    L.set_option('lanes', 1)
    L.set_profiling(True)
    out = {}
    try:
        for name, fn in (('prove', case.prove_dev), ('verify', case.verify_dev)):
            L.profile_reset()
            fn()
            torch.cuda.synchronize()
            prof = L.profile()
            total = sum(v['ms'] for v in prof.values())
            tasks = {t: next((v for k, v in prof.items() if k.endswith(t)), None) for t in GK_TASKS}
            out[name] = {'all_kernels_ms': total,
                         'tasks': {t: {'ms': v['ms'], 'launches': v['launches'], 'share_of_kernel_ms': v['ms'] / total}
                                   for t, v in tasks.items() if v}}
    finally:
        L.set_profiling(False)
        L.set_option('lanes', lanes)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='write the whole record here as JSON')
    a = ap.parse_args()
    L = ZkaLib(device=0)
    hn, hp = L.params_generate(synth.params_rnd(0))
    P = L.params_create(hn, hp, SEC)
    out = {'card': card(), 'lanes': L.config()['lanes'], 'sec_level': SEC, 'samples': K, 'rows': B, 'cases': {}}
    sizes = [8 << (i % 8) for i in range(64)]
    depth = [VT.ceil_log2(s) for s in sizes]
    grouped = np.array(sorted((b % 64 for b in range(B)), key=lambda r: (depth[r], r)), np.uint32)
    wb = synth.RingsWorkload(B, sizes, grouped, seed=2)
    first = {r: np.flatnonzero(grouped == r) for r in range(64)}
    il_rows = np.array([int(first[b % 64][b // 64]) for b in range(B)])       # round-robin over the rings: a new depth per row
    cg, ci = TapeCase(L, P, wb), TapeCase(L, P, wb, il_rows)
    assert all(depth[int(x)] != depth[int(y)] for x, y in zip(ci.ring_of, ci.ring_of[1:]))
    wa = synth.RingsWorkload(B, [8] * B, np.arange(B), seed=1)
    ca = Case(L, P, wa)
    cases = {'mixed64_grouped': of_case(cg, True), 'mixed64_interleaved': of_case(ci, True), 'own8': of_case(ca, False),
             'config1': config1(L, P)}
    kinds = ('prove_dev', 'verify_dev', 'prove_tape', 'verify_tape')
    rates = {n: {k: [] for k in kinds if k in c} for n, c in cases.items()}
    for rnd in range(4):                                  # round 0 warms every shape up
        for n, c in cases.items():
            for k in rates[n]:
                t = timed(c[k])
                if rnd:
                    rates[n][k].append(c['rows'] / t)
            c['check']()
    # the seeded proofs (the last prove of each case was the tape one: prove once more), row by row
    cg.prove_dev()
    ci.prove_dev()
    sg, si = cg.checksums(), ci.checksums()
    same = all(si[i] == sg[int(b)] for i, b in enumerate(il_rows))
    assert same
    cg.prove_tape()
    ci.prove_tape()
    tape_same = cg.checksums() == sg and ci.checksums() == si
    assert tape_same
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    for n in cases:
        out['cases'][n] = {'rows': cases[n]['rows'], 'rates_per_s': rates[n], 'median_per_s': {k: med(v) for k, v in rates[n].items()}}
        print(json.dumps({'case': n, **out['cases'][n]}), flush=True)
    out['proofs_equal_interleaved_vs_grouped'] = bool(same)
    out['proofs_equal_tape_vs_seeded'] = bool(tape_same)
    out['checksum_of_checksums'] = hashlib.sha256(''.join(sg).encode()).hexdigest()
    out['gk_profile'] = {'mixed64_grouped': gk_profile(L, cg), 'mixed64_interleaved': gk_profile(L, ci)}
    print(json.dumps({'gk_profile': out['gk_profile']}), flush=True)
    for c in (cg, ci, ca):
        c.close()
    L.params_destroy(P)
    out['card_after'] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps({'card': out['card'], 'proofs_equal_interleaved_vs_grouped': bool(same)}))


if __name__ == '__main__':
    main()
