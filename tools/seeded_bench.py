"""Tape mode against seeded mode (randomness expanded on the GPU from 32 bytes per proof), in one process.

For each workload (config2: 8192 proofs, ring 256; config1: 1024 proofs, ring 8; SecLevel 80): warm-up, then three
rounds that alternate the two modes, each timed with a device synchronise at its end:
  * device-resident prove and verify (inputs, seeds / tapes and outputs in HBM);
  * host-buffer end-to-end prove: tape mode without and with making the tape on the host (api.synth_os_tape), seeded
    mode with os.urandom seeds;
then one profiled pass per mode for the expansion kernels' time (zka_profile_json), the host-to-device bytes a
host-buffer step moves, and a checksum showing seeded proofs equal tape-mode proofs on the expanded tapes.

    python tools/seeded_bench.py [--out FILE.json] [--workloads config2,config1]

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

from zkp_ecdsa_b200 import api, synth  # noqa: E402

SEC = 80
K = 20
WORKLOADS = {'config1': (1024, 8), 'config2': (8192, 256)}


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


def run(eng, wname):
    B, N = WORKLOADS[wname]
    L = eng.lib
    params = eng.generate_params_list(SEC, rnd=synth.params_rnd(0))
    P = params.handle
    wl = synth.Workload(B, N, seed=0, distinct_signers=min(B, N))
    n = (N - 1).bit_length()
    ts, vts, ps = L.prove_tape_len(N, SEC), L.verify_tape_len_ex(N, SEC, K), L.proof_max_len(N, SEC)
    seeds = np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32).copy()
    vseeds = np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32).copy()
    tape = L.seed_tape(0, seeds, N, SEC)               # tape mode runs on the tapes the seeds stand for
    vtape = L.seed_tape(1, vseeds, N, SEC, K)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    d_msg, d_sig, d_pk, d_which, d_ring = dev(wl.msg_hash), dev(wl.sig), dev(wl.pk), dev(wl.which.view(np.int32)), dev(wl.ring)
    d_seed, d_vseed, d_tape, d_vtape = dev(seeds), dev(vseeds), dev(tape), dev(vtape)
    d_pr = {m: torch.zeros(B * ps, dtype=torch.uint8, device='cuda') for m in ('tape', 'seeded')}
    d_len = {m: torch.zeros(B, dtype=torch.int32, device='cuda') for m in ('tape', 'seeded')}
    d_st = torch.zeros(B, dtype=torch.int32, device='cuda')
    d_ok = torch.zeros(B, dtype=torch.uint8, device='cuda')
    ptr = lambda t: t.data_ptr()   # noqa: E731

    def prove_dev(m):
        if m == 'tape':
            L.prove_batch(P, B, ptr(d_msg), ptr(d_sig), ptr(d_pk), ptr(d_which), ptr(d_ring), N, ptr(d_tape), ts, ptr(d_pr[m]), ps,
                          ptr(d_len[m]), ptr(d_st))
        else:
            L.prove_batch_seeded(P, B, ptr(d_msg), ptr(d_sig), ptr(d_pk), ptr(d_which), ptr(d_ring), N, ptr(d_seed), ptr(d_pr[m]), ps,
                                 ptr(d_len[m]), ptr(d_st))

    def verify_dev(m):
        if m == 'tape':
            L.verify_batch_ex(P, B, ptr(d_msg), ptr(d_ring), N, ptr(d_pr['tape']), ps, ptr(d_len['tape']), ptr(d_vtape), vts,
                              ptr(d_ok), ptr(d_st), K)
        else:
            L.verify_batch_seeded(P, B, ptr(d_msg), ptr(d_ring), N, ptr(d_pr['tape']), ps, ptr(d_len['tape']), ptr(d_vseed), K,
                                  ptr(d_ok), ptr(d_st))

    h_pr = np.zeros((B, ps), np.uint8)
    h_len = np.zeros(B, np.uint32)
    h_st = np.zeros(B, np.int32)

    def e2e(m):
        if m == 'tape':
            L.prove_batch(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, tape, ts, h_pr, ps, h_len, h_st)
        elif m == 'tape+hostgen':
            t = api.synth_os_tape(B, ts, SEC)
            L.prove_batch(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, t, ts, h_pr, ps, h_len, h_st)
        else:
            s = np.frombuffer(os.urandom(32 * B), np.uint8).reshape(B, 32)
            L.prove_batch_seeded(P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, s, h_pr, ps, h_len, h_st)

    for m in ('tape', 'seeded'):                       # warm-up of every shape
        prove_dev(m)
        verify_dev(m)
        e2e(m)
    e2e('tape+hostgen')
    res = {'prove_dev': {'tape': [], 'seeded': []}, 'verify_dev': {'tape': [], 'seeded': []},
           'prove_e2e': {'tape': [], 'tape+hostgen': [], 'seeded': []}}
    for _ in range(3):
        for m in ('tape', 'seeded'):
            res['prove_dev'][m].append(B / timed(lambda: prove_dev(m)))
            res['verify_dev'][m].append(B / timed(lambda: verify_dev(m)))
        for m in ('tape', 'tape+hostgen', 'seeded'):
            res['prove_e2e'][m].append(B / timed(lambda: e2e(m)))
        assert not d_st.cpu().numpy().any() and d_ok.cpu().numpy().all()
    # equality at the timed size: seeded proofs against tape-mode proofs on the expanded tapes
    prove_dev('tape')
    prove_dev('seeded')
    torch.cuda.synchronize()
    sums = {m: hashlib.sha256(d_pr[m].cpu().numpy().tobytes() + d_len[m].cpu().numpy().tobytes()).hexdigest() for m in d_pr}
    assert sums['tape'] == sums['seeded'], sums
    # H2D bytes of one host-buffer prove step: the per-proof rows, then the tape as it travels (the 3 + 4S draws up front,
    # the item / GK draws up to the longest proof of each chunk) or 32 seed bytes
    plen = d_len['tape'].cpu().numpy().astype(np.int64)
    gk = 1 + 4 * n * L.wp + (3 * n + 1) * L.ws
    z = (plen - 2 * 65 - 2 * L.wp - SEC * L.rep1_len - gk) // (L.rep0_len - L.rep1_len)
    off = L.chunk_schedule(B, host_buffers=True)
    rows = B * (32 + 64 + 65 + 4)
    tape_h2d = sum((off[k + 1] - off[k]) * 32 * (3 + 4 * SEC + 40 * int(z[off[k]:off[k + 1]].max()) + 5 * n) for k in range(len(off) - 1))
    h2d = {'tape': rows + tape_h2d, 'seeded': rows + 32 * B}
    # kernel time of the expansion, in a profiled pass of its own
    L.set_profiling(True)
    L.profile_reset()
    prove_dev('seeded')
    verify_dev('seeded')
    torch.cuda.synchronize()
    prof = L.profile()
    L.set_profiling(False)
    exp_ms = {k.split('::')[-1]: v for k, v in prof.items() if 'Seed' in k}
    total_ms = sum(v['ms'] for v in prof.values())
    params.close()
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    return {'workload': wname, 'B': B, 'N': N, 'sec_level': SEC, 'samples': K,
            'rates_per_s': res,
            'median_per_s': {k: {m: med(v) for m, v in d.items()} for k, d in res.items()},
            'h2d_bytes_per_step': h2d, 'expansion_kernels': exp_ms, 'profiled_kernel_ms_total': total_ms,
            'checksum_seeded_equals_tape': sums['seeded']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='write the whole record here as JSON')
    ap.add_argument('--workloads', default='config2,config1')
    a = ap.parse_args()
    eng = api.Engine(0)
    out = {'card': card(), 'lanes': eng.lib.config()['lanes'], 'runs': []}
    for w in a.workloads.split(','):
        r = run(eng, w)
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
