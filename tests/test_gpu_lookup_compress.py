"""mv_lookup::Argument::prepare's compression with theta on the device: DeviceOps::compress_expressions runs keygen's compression
programs through b200zk_graph_evaluate (log_size = k, rot_scale = 1) on the Lagrange columns, each read column uploaded once.

- bit-exact against the host default of Ops::compress_expressions and the oracle's interpreter, for k = 1 .. 24, with the
  generator of tests/test_lookup_compress_oracle.py; up to k = 10 also against the big-integer fold;
- create_proof on the device with every compression checked against the host default, on the three session circuits (the
  two-phase circuit's challenge-combined lookup, the wide circuit's two-term input), whole-coset keys and keys without cosets;
- column tables with entries no program reads, and a program reading a column that was not supplied (B200ZK_E_INVALID).
"""
import hashlib
import json
import subprocess

import numpy as np
import pytest

from lookup_compress_model import every_kind
from lookup_model import small_ints
from oracle import oracle as O
from test_lookup_compress_oracle import DIGESTS, SHAPE, binary, model, random_case
from lookup_compress_model import write_case
from test_plonk_session import GPU_CASES, key


def run(*args, timeout=1800):
    r = subprocess.run([binary()] + [str(a) for a in args], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def selector_case(k):
    """(q a, q b, q a(omega X)) with a 0/1 selector q: an inner-circuit lookup input"""
    n = 1 << k
    q = small_ints((np.arange(n) % 3 == 0).astype(np.int64))
    a, b = O.fill_fr(n, 71), O.fill_fr(n, 72)
    side = [("mul", ("fixed", 0, 0), ("advice", 0, 0)), ("mul", ("fixed", 0, 0), ("advice", 1, 0)),
            ("mul", ("fixed", 0, 0), ("advice", 0, 1))]
    return 12345, [], [q], [a, b], [], [side]


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 5, 10, 16, 20, 24])
def test_device_equals_host_default_and_oracle(tmp_path, k):
    if k == 24:
        case = selector_case(k)
    else:
        case = random_case(100 + k, k, [1, 2, 3, 4] if k <= 10 else [3, 2])
        case[5].append(every_kind(SHAPE))
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    write_case(src, k, *case)
    out = run("device", src, dst if k <= 10 else "-")
    assert "device == host default == oracle interpreter" in out
    if k <= 10:
        got = np.fromfile(dst, np.uint64).reshape(len(case[5]), 1 << k, 4)
        for s, want in enumerate(model(k, case)):
            assert np.array_equal(got[s], want), s


@pytest.mark.gpu
@pytest.mark.parametrize("k,seed,variant", GPU_CASES)
def test_session_compression_on_the_device_equals_the_host_default(k, seed, variant):
    out = run("session_device", k, seed, variant)
    assert "device compression == host default" in out
    proofs = {l.split()[1]: bytes.fromhex(l.split()[2]) for l in out.splitlines() if l.startswith("proof_sha_input")}
    assert proofs["device_whole"] == proofs["device_parts"]
    digests = json.load(open(DIGESTS))
    if key(k, seed, variant) in digests:
        assert hashlib.sha256(proofs["device_whole"]).hexdigest() == digests[key(k, seed, variant)]


@pytest.mark.gpu
def test_column_tables_with_unreferenced_entries_and_a_missing_column():
    out = run("tables")
    assert "unreferenced entries: device == host default on 3 sides" in out
    why = [l for l in out.splitlines() if l.startswith("column not supplied ->")][0]
    assert "b200zk error -1" in why and "the program reads fixed/advice/instance columns up to 7" in why, why
