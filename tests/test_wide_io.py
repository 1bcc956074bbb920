"""16-byte transactions of the prover: tape draws read as two 16-byte loads when 16-byte aligned, 80-byte encoding
slots, and the ByteWriter that writes proof regions of any alignment with 16-byte stores.  None of it may change a
byte: every tape base offset and stride, host or device tape, odd proof stride and misaligned output base gives the
proofs of the aligned default, whose spot rows match the oracle."""
import os
import subprocess
import textwrap

import numpy as np
import pytest

import common
from zkp_ecdsa_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'zkp_ecdsa_b200', 'csrc')
SEC, B, N = 12, 3, 6


def _rows(flat_buf, off, rows, stride):
    """rows x stride view starting `off` bytes into a 1-D buffer (a misaligned base for a C caller)"""
    return flat_buf[off:off + rows * stride].reshape(rows, stride)


def _host_tape(tape, off, stride):
    buf = np.zeros(off + tape.shape[0] * stride + 16, np.uint8)
    v = _rows(buf, off, tape.shape[0], stride)
    v[:, :tape.shape[1]] = tape
    return v


class Prover:
    """prove_batch with caller-chosen tape and proof-row placement; returns the proofs as [B][proof_len] bytes"""

    def __init__(self, L, gpu):
        self.L, self.gpu = L, gpu
        self.P, self.po = common.make_params(L, 5, SEC)
        self.wl = synth.Workload(B=B, N=N, seed=5)
        self.ts = L.prove_tape_len(N, SEC)
        self.tape = synth.random_tape(B, self.ts, seed=105)
        self.ps = L.proof_max_len(N, SEC)

    def run(self, tape_ptr, stride, proof_stride=None, out_off=0, dev_out=False):
        L, wl = self.L, self.wl
        ps = proof_stride or self.ps
        plen = np.zeros(B, np.uint32)
        st = np.zeros(B, np.int32)
        if dev_out:
            import torch
            buf = torch.zeros(out_off + B * ps + 16, dtype=torch.uint8, device='cuda')
            L.prove_batch(self.P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, tape_ptr, stride,
                          buf.data_ptr() + out_off, ps, plen, st)
            torch.cuda.synchronize()
            rows = _rows(buf.cpu().numpy(), out_off, B, ps)
        else:
            buf = np.zeros(out_off + B * ps + 16, np.uint8)
            rows = _rows(buf, out_off, B, ps)
            L.prove_batch(self.P, B, wl.msg_hash, wl.sig, wl.pk, wl.which, wl.ring, N, tape_ptr, stride, rows, ps, plen, st)
        assert (st == 0).all(), st
        return [rows[b, :plen[b]].tobytes() for b in range(B)]

    def host(self, off, stride, **kw):
        return self.run(_host_tape(self.tape, off, stride), stride, **kw)

    def device(self, off, stride, **kw):
        import torch
        t = torch.from_numpy(_host_tape(self.tape, 0, stride).reshape(-1).copy())
        d = torch.zeros(off + t.numel() + 16, dtype=torch.uint8, device='cuda')
        d[off:off + t.numel()].copy_(t)
        return self.run(d.data_ptr() + off, stride, **kw)


def check_prove_placements(L, gpu):
    pv = Prover(L, gpu)
    ref = pv.host(0, pv.ts)
    for b in (0, B - 1):                                          # spot rows against the oracle
        pr, _ = common.oracle_proof(pv.po, pv.wl, pv.tape, b)
        assert ref[b] == common.flat.ser_proof(pr), b
    ts = pv.ts
    assert ts % 16 == 0
    for off, stride in ((1, ts + 4), (4, ts + 8), (0, ts + 4), (12, ts)):   # host tapes: staged at a 16-byte pitch
        assert pv.host(off, stride) == ref, ('host tape', off, stride)
    # proof rows at an odd stride from a misaligned base
    assert pv.host(0, ts, proof_stride=pv.ps + 3, out_off=5) == ref
    if gpu:
        for off in (1, 4, 8, 12):
            for stride in (ts, ts + 4, ts + 8):
                assert pv.device(off, stride) == ref, ('device tape', off, stride)
        assert pv.device(0, ts, proof_stride=pv.ps + 1, out_off=7, dev_out=True) == ref
        assert pv.device(4, ts + 4, proof_stride=pv.ps + 3, out_off=3, dev_out=True) == ref
    L.params_destroy(pv.P)


def _misaligned(tape, off=3, extra=4):
    """the same draws from a base `off` bytes past a 16-byte boundary, rows `extra` bytes longer"""
    return _host_tape(tape, off, tape.shape[1] + extra)


def check_standalone_misaligned(L):
    """the stand-alone provers give the same bytes for a misaligned tape (rows not on 16-byte boundaries)"""
    P, _ = common.make_params(L, 81, 8)
    tom = common.pg(L)
    d = synth.Drbg(81, 'wide')
    q = tom.order
    i32 = lambda v: int(v).to_bytes(32, 'big')   # noqa: E731
    arr = lambda rr: np.array([list(x) for x in rr], np.uint8)   # noqa: E731
    for kind, nd, ns in (('equality', 3, 3), ('mult', 7, 6)):
        tape = synth.random_tape(B, 32 * nd, seed=82)
        if kind == 'equality':
            rows = [i32(x) + i32(d.below(q)) + i32(d.below(q)) for x in (d.below(q) for _ in range(B))]
        else:
            rows = []
            for _ in range(B):
                x, y = d.below(q), d.below(q)
                rows.append(i32(x) + i32(y) + i32(x * y % q) + b''.join(i32(d.below(q)) for _ in range(3)))
        a = L.prove_sub_batch(kind, P, arr(rows), tape)
        for extra in (4, 8, 12):
            b_ = L.prove_sub_batch(kind, P, arr(rows), _misaligned(tape, 3, extra))
            assert all((x == y).all() for x, y in zip(a, b_)), (kind, extra)
    # pointadd: P + Q = R
    from oracle.curves import p256
    pts, bl = [], synth.random_tape(B, 32 * 6, seed=83)
    for _ in range(B):
        Pp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        Qp = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        pts.append(common.flat._pt(Pp, 65) + common.flat._pt(Qp, 65) + common.flat._pt(Pp.add(Qp), 65))
    tape = synth.random_tape(B, 32 * 38, seed=84)
    a = L.prove_sub_batch('pointadd', P, arr(pts), tape, bl)
    assert (a[2] == 0).all()
    b_ = L.prove_sub_batch('pointadd', P, arr(pts), _misaligned(tape, 5, 4), bl)
    assert all((x == y).all() for x, y in zip(a, b_))
    # membership: internal rows of 96 + stride bytes, rounded up to a multiple of 16
    ring = np.array([list(int(v).to_bytes(32, 'big')) for v in (3, 5, 7, 11, 13)], np.uint8)
    rs = synth.random_tape(B, 32, seed=85)
    idx = np.array([3, 0, 4], np.uint32)
    tape = synth.random_tape(B, 32 * 5 * 3, seed=86)
    a = L.prove_membership_batch(P, rs, idx, ring, tape)
    assert (a[2] == 0).all()
    for extra in (4, 8):
        b_ = L.prove_membership_batch(P, rs, idx, ring, _misaligned(tape, 1, extra))
        assert all((x == y).all() for x, y in zip(a, b_)), extra
    L.params_destroy(P)
    # proveExp alone (tape layout of zka_prove_batch, rows of the repetitions only)
    P, _ = common.make_params(L, 87, 6)
    base, s_, pk = [], [], []
    for _ in range(B):
        g = p256.generator().mul(p256.new_scalar(d.below(p256.order)))
        s = d.below(p256.order)
        base.append(common.flat._pt(g, 65)); s_.append(i32(s)); pk.append(common.flat._pt(g.mul(p256.new_scalar(s)), 65))
    tape = synth.random_tape(B, 32 * (3 + 44 * 6), seed=88)
    a = L.prove_exp_batch(P, arr(base), arr(s_), arr(pk), None, tape, 6)
    assert (a[2] == 0).all()
    b_ = L.prove_exp_batch(P, arr(base), arr(s_), arr(pk), None, _misaligned(tape, 3, 4), 6)
    assert all((x == y).all() for x, y in zip(a, b_))
    L.params_destroy(P)


def test_prove_placements_hostsim(hostsim):
    check_prove_placements(hostsim, False)


def test_prove_placements_hostsim_war(hostsim_war):
    check_prove_placements(hostsim_war, False)


def test_standalone_misaligned_hostsim(hostsim):
    check_standalone_misaligned(hostsim)


def test_standalone_misaligned_hostsim_war(hostsim_war):
    check_standalone_misaligned(hostsim_war)


@pytest.mark.gpu
def test_prove_placements_on_gpu(gpu_engine):
    check_prove_placements(gpu_engine.lib, True)


@pytest.mark.gpu
def test_prove_placements_on_gpu_war(gpu_engine_war):
    check_prove_placements(gpu_engine_war.lib, True)


@pytest.mark.gpu
def test_standalone_misaligned_on_gpu(gpu_engine):
    check_standalone_misaligned(gpu_engine.lib)


@pytest.mark.gpu
def test_standalone_misaligned_on_gpu_war(gpu_engine_war):
    check_standalone_misaligned(gpu_engine_war.lib)


# ----------------------------------------------------------------------------------------- the ByteWriter alone
_WRITER_HARNESS = textwrap.dedent('''
    #include "zk_ops.cuh"
    using namespace zk;
    // regions of `len` pieces each: piece kinds 0 = byte, 1 = 33-byte scalar, 2 = 32-byte scalar, 3 = 67-byte point
    extern "C" void write_regions(uint8_t* buf, const int* starts, int nreg, const int* kinds, int npieces,
                                  const uint8_t* slots, const uint32_t* scalars) {
      for (int r = 0; r < nreg; r++) {
        ByteWriter o(buf + starts[r]);
        for (int i = 0; i < npieces; i++) {
          const int k = kinds[(r + i) % npieces];
          if (k == 0) o.put_byte(scalars[8 * i] & 0xffu);
          else if (k == 1) o.put_scalar<33>(scalars + 8 * i);
          else if (k == 2) o.put_scalar<32>(scalars + 8 * i);
          else o.put_point<67>(slots + (size_t)BSTRIDE * i);
        }
        o.finish();
      }
    }
''')
_FLUSH = 'if (lead == 0) st4(blk, q); else store_part(lead, 16);'


def _build_writer(tmp, mutate):
    src_dir = os.path.join(tmp, 'mut' if mutate else 'orig')
    os.makedirs(src_dir)
    for f in os.listdir(CSRC):
        if f.endswith(('.cuh', '.h', '.inc')):
            s = open(os.path.join(CSRC, f)).read()
            if f == 'zk_ops.cuh':
                assert _FLUSH in s
                if mutate:   # the first block of a region written whole: clobbers the preceding region's bytes
                    s = s.replace(_FLUSH, 'st4(blk, q);')
            open(os.path.join(src_dir, f), 'w').write(s)
    open(os.path.join(src_dir, 'h.cc'), 'w').write(_WRITER_HARNESS)
    out = os.path.join(src_dir, 'libw.so')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-DZKA_HOSTSIM', '-x', 'c++', '-I' + os.path.join(ROOT, 'include'),
                           '-I' + src_dir, '-fPIC', '-shared', '-o', out, os.path.join(src_dir, 'h.cc')])
    return out


def _writer_ok(lib_path):
    """every alignment of a region start, regions back to back and with gaps: the region bytes are the expected
    stream and no byte outside the regions changes"""
    import ctypes as C
    lib = C.CDLL(lib_path)
    rng = np.random.default_rng(7)
    npieces = 7
    kinds = np.array([0, 1, 3, 2, 3, 1, 0], np.int32)
    lens = {0: 1, 1: 33, 2: 32, 3: 67}
    slots = np.zeros(npieces * 80, np.uint8)
    pts = [rng.integers(0, 256, 67, dtype=np.uint8) for _ in range(npieces)]
    for i, p in enumerate(pts):
        slots[80 * i:80 * i + 67] = p
        slots[80 * i + 67:80 * i + 80] = 0xee               # slot padding must never reach the output
    sc = rng.integers(0, 2 ** 32, (npieces, 8), dtype=np.uint64).astype(np.uint32)
    sc[:, 7] &= 0x7fffffff

    def piece(k, i):
        if k == 0:
            return bytes([int(sc[i, 0]) & 0xff])
        if k in (1, 2):
            v = sum(int(sc[i, j]) << (32 * j) for j in range(8))
            return v.to_bytes(lens[k], 'big')
        return pts[i].tobytes()

    for first in range(16):
        for gap in (0, 1, 5):
            stream = [b''.join(piece(int(kinds[(r + i) % npieces]), i) for i in range(npieces)) for r in range(3)]
            starts, pos = [], 16 + first
            for s in stream:
                starts.append(pos)
                pos += len(s) + gap
            buf = np.full(pos + 32, 0xa5, np.uint8)
            want = buf.copy()
            for st, s in zip(starts, stream):
                want[st:st + len(s)] = np.frombuffer(s, np.uint8)
            lib.write_regions(buf.ctypes.data_as(C.c_void_p), np.array(starts, np.int32).ctypes.data_as(C.c_void_p), 3,
                              kinds.ctypes.data_as(C.c_void_p), npieces, slots.ctypes.data_as(C.c_void_p),
                              sc.ctypes.data_as(C.c_void_p))
            if not (buf == want).all():
                return False
    return True


def test_byte_writer_regions_and_mutation(tmp_path):
    """The writer's output at every alignment is the byte stream with its neighbours intact; a writer that stores the
    region's first block whole (clobbering the bytes of the region before it) is caught."""
    assert _writer_ok(_build_writer(str(tmp_path), False))
    assert not _writer_ok(_build_writer(str(tmp_path), True))
