"""CPU-only: the port of RocksDB's StringAppendOperator (tests/string_append_model.py) against what the reference's
RocksDB binary answered on the recorded streams (tests/golden/string_append.json), and against the live binary on
seeded random streams when oracle/_ref is built."""
import shutil

import pytest

import string_append_oracle as O
from oracle import okv

CASES = O.load_cases()
NAMES = sorted(O.cases())


def test_fixture_covers_every_case():
    assert sorted(CASES) == NAMES


@pytest.mark.parametrize("name", NAMES)
def test_port_matches_recorded_reference(name):
    delim, steps = O.cases()[name]
    assert O.run_case(O.ModelSide(delim), steps) == CASES[name]


@pytest.mark.skipif(not okv.ref_available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("seed", range(12))
def test_port_matches_live_reference(seed):
    delim = [b",", None, b"\0", b"|"][seed % 4]
    steps = O._stream(50000 + seed)
    ref = O.RefSide(delim)
    try:
        got = O.run_case(ref, steps)
    finally:
        ref.close()
        shutil.rmtree(ref.db._tmp, ignore_errors=True)
    assert O.run_case(O.ModelSide(delim), steps) == got
