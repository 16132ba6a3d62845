#!/usr/bin/env python
"""Generate tests/golden/doubles.json from the UNMODIFIED reference (oracle/_ref/libsj_ref_double.so): get_double vectors.

For every text of tests/test_double_oracle.py's golden_texts() (the named cases of tests/double_cases.py and 2 000
seeded numbers), the reference's error and the double's bits (hex) for the document [text] at /0.  Written only after
the oracle (sjo_double) and Python's float() were found to agree.

    python oracle/gen_golden_doubles.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import double_cases as DC  # noqa: E402
import double_oracle as DO  # noqa: E402
import test_double_oracle as T  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "doubles.json")


def main():
    ref, dbl = DO.RefDoubles(), DO.Doubles()
    cases = []
    for t in T.golden_texts():
        e, b = ref.of_text(t)
        assert (e, b) == DC.expect(t) and dbl.of_text(t)[::2] == (e, b), t[:60]
        cases.append([int(e), f"{b:016x}"])
    json.dump({"generator": "oracle/gen_golden_doubles.py", "cases": cases}, open(OUT, "w"))
    print(len(cases), "numbers ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
