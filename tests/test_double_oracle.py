"""The get_double oracle (sjo_double, oracle/sj_double_oracle.c) pinned to the reference's element::get_double after
dom::parser::parse and at_pointer, and both to Python's float() (correctly rounded), bit for bit: the edge cases of
tests/double_cases.py (Clinger boundaries, halfway points written out, subnormals, the largest double, infinities,
zeros, exponents of more than 18 digits, a 10 000-digit mantissa, integers) and seeded numbers.  Without the
reference, the oracle and float() against tests/golden/doubles.json."""
import json
import os

import pytest

import double_cases as DC
import double_oracle as DO
import oracle_lib as O

GOLDEN = os.path.join(O.ROOT, "tests", "golden", "doubles.json")


def golden_texts():
    return DC.named_cases() + DC.random_numbers(2000, 11)


def check(texts, want_of):
    dbl = DO.Doubles()
    for t in texts:
        we, wb = want_of(t)
        e, rt, b = dbl.of_text(t)
        fe, fb = DC.expect(t)
        assert (e, b) == (we, wb) == (fe, fb), (t[:60], e, hex(b), we, hex(wb), fe, hex(fb))
        want_type = (ord("u") if int(t) > 2 ** 63 - 1 else ord("l")) if DC.is_integer(t) else ord("d")
        assert rt == want_type, (t[:60], rt)


@pytest.mark.skipif(not DO.have_ref(), reason="reference build (oracle/_ref) not present")
def test_oracle_and_float_match_reference():
    ref = DO.RefDoubles()
    check(golden_texts() + DC.slow_heavy(500, 3), ref.of_text)


def test_oracle_and_float_match_golden():
    g = json.load(open(GOLDEN))
    texts = golden_texts()
    assert len(g["cases"]) == len(texts)
    want = {}
    for t, (e, b) in zip(texts, g["cases"]):
        want[t] = (e, int(b, 16))
    check(texts, lambda t: want[t])
