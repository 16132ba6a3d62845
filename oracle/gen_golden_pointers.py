#!/usr/bin/env python
"""Generate tests/golden/pointers.json from the UNMODIFIED reference (oracle/_ref/libsj_ref_pointer.so, with oracle/_ref/libsj_ref.so for the round trip): JSON Pointer vectors.

For every case of tests/pointer_cases.py (reduced: twitter up to depth 3, citm up to depth 2) the reference's
dom::element::at_pointer error, and on success the byte offset at which the selected value starts.  The offset is the
oracle's (sjo_at_pointer), written only after the raw span it names, parsed and minified by the reference, was found equal
to the reference's serialisation of the element.

    python oracle/gen_golden_pointers.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib as O  # noqa: E402
import pointer_oracle as PO  # noqa: E402
import pointer_cases as PC  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "pointers.json")


def main():
    port, ref, rp = PO.Pointers(), O.Ref(), PO.RefPointers()
    cases = []
    for name, doc, pointers in PC.corpus_cases(full=False):
        r, tw, _s, err, idx = port.table(doc, pointers)
        want = rp.at_pointer(doc, pointers)
        byte = []
        for p, (werr, wval) in enumerate(want):
            assert err[p, 0] == werr, (name, pointers[p])
            if werr == 0:
                assert ref.dom_roundtrip(PO.value_span(doc, r.idx, tw[1], idx[p, 0]))[1] == wval, (name, pointers[p])
            byte.append(int(r.idx[idx[p, 0]]) if werr == 0 else -1)
        ent = {"file": name} if name.endswith(".json") else {"doc": doc.hex()}
        ent.update({"pointers": pointers, "err": [int(w[0]) for w in want], "byte": byte})
        cases.append(ent)
    json.dump({"generator": "oracle/gen_golden_pointers.py", "cases": cases}, open(OUT, "w"))
    print(sum(len(c["pointers"]) for c in cases), "pointers ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
