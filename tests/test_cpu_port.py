"""oracle/cpu (C++ restatement of the reference algorithms, baseline + fast checker) against the Python oracle
and the committed golden fixtures.  Both are test infrastructure; the product never loads either."""
import numpy as np
import pytest

import common
from zkp_ecdsa_b200 import synth


@pytest.fixture(scope='module')
def cpu_port():
    import __graft_entry__ as g
    g.build_oracle_cpu()
    from zkp_ecdsa_b200.capi import ZkaLib
    return ZkaLib(g.ORACLE_CPU)


def test_layers(cpu_port):
    common.check_field_ops(cpu_port, count=40)
    common.check_hash(cpu_port)
    common.check_p256_mul(cpu_port, count=4)
    P, po = common.make_params(cpu_port, seed=5)
    common.check_tom_commit(cpu_port, P, po, count=4)
    cpu_port.params_destroy(P)


def test_whole_proof_bytes_equal_python_oracle(cpu_port):
    common.check_prove_parity(cpu_port, B=1, N=6, seed=3, sec_level=80)
    common.check_prove_parity(cpu_port, B=2, N=17, seed=4, sec_level=16)     # ragged ring


def test_verify_decisions_equal_python_oracle(cpu_port):
    # 16 random tampers + the 2 non-canonical point encodings
    assert common.check_verify_parity(cpu_port, N=6, seed=3, tampers=16, sec_level=20) == 18


@pytest.mark.parametrize('tag', ['a', 'b', 'c', 'd'])
def test_golden(cpu_port, tag):
    import test_golden as TG
    TG._check_lib(cpu_port, tag)


def test_error_statuses_and_rows(cpu_port):
    L = cpu_port
    P, _ = common.make_params(L, 31, 16)
    wl = synth.Workload(B=4, N=8, seed=31)
    tape = synth.random_tape(4, L.prove_tape_len(8, 16), seed=32)
    wl.pk[1, 40] ^= 1
    wl.which[2] = 0xFFFFFFFF
    tape[3, 32 * 3:32 * 3 + 4] = 255
    proofs, plen, status = common.run_prove(L, P, wl, tape, 16)
    assert list(status) == [0, 1, 6, 5]
    assert plen[0] > 0 and not plen[1:].any() and not proofs[1:].any()
    L.params_destroy(P)


def test_threads_give_identical_results(cpu_port, monkeypatch):
    import __graft_entry__ as g
    from zkp_ecdsa_b200.capi import ZkaLib
    monkeypatch.setenv('ZKA_CPU_THREADS', '4')
    L4 = ZkaLib(g.ORACLE_CPU)
    P1, _ = common.make_params(cpu_port, 9, 16)
    P4, _ = common.make_params(L4, 9, 16)
    wl = synth.Workload(B=6, N=5, seed=9)
    tape = synth.random_tape(6, cpu_port.prove_tape_len(5, 16), seed=10)
    a = common.run_prove(cpu_port, P1, wl, tape, 16)
    b = common.run_prove(L4, P4, wl, tape, 16)
    assert (a[1] == b[1]).all() and (a[0] == b[0]).all() and not a[2].any()


@pytest.mark.parametrize('K', [5, 33])
def test_verify_sample_count_cpu_port_vs_python(cpu_port, K):
    """verifyExp's secparam as a parameter: the C++ port against the Python oracle."""
    common.check_verify_samples(cpu_port, K, N=5, seed=15, sec_level=40, tampers=2, oracle='python')
