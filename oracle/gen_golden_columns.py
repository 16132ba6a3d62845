#!/usr/bin/env python
"""Generate tests/golden/columns.json from the UNMODIFIED reference (oracle/_ref/libsj_ref_column.so): typed-column vectors.

For every document of tests/column_cases.py and every getter kind (get_int64, get_uint64, get_bool, get_string,
get_array().size(), get_object().size()), the reference's error for each pointer after at_pointer, and on success the
value (as a decimal string) or the string's bytes (hex).  Written only after the oracle (sjo_column) was found to agree.

    python oracle/gen_golden_columns.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import column_cases as CC  # noqa: E402
import column_oracle as CO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "columns.json")


def reference_vectors(ref, kind, doc, pointers):
    _perr, res = ref.column(kind, doc, pointers)
    return {"err": [int(e) for e, _v, _s in res], "value": [str(int(v)) for _e, v, _s in res], "bytes": [s.hex() for _e, _v, s in res]}


def main():
    cols, ref = CO.Columns(), CO.RefColumns()
    cases = []
    for name, doc, pointers in CC.documents():
        ent = {"name": name, "pointers": pointers, "kinds": {}}
        if not name.startswith(("long", "row")):  # those are rebuilt by tests/column_cases.py
            ent["doc"] = doc.hex()
        for kind in CO.KINDS:
            want = reference_vectors(ref, kind, doc, pointers)
            _tab, err, _rt, val, strs = cols.of_document(kind, doc, pointers)
            assert err[:, 0].tolist() == want["err"], (name, kind)
            if kind == CO.STRING:
                assert [s.hex() for s in strs] == want["bytes"], (name, kind)
                del want["value"]
            else:
                assert [str(int(v)) for v in val[:, 0]] == want["value"], (name, kind)
                del want["bytes"]
            ent["kinds"][str(kind)] = want
        cases.append(ent)
    json.dump({"generator": "oracle/gen_golden_columns.py", "cases": cases}, open(OUT, "w"))
    print(len(cases), "documents ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
