"""Writes tests/golden/document_errors.json: the verdicts of stage 2 (error, structural index) for the grammar cases,
streams and depth cases, from the grammar oracle (oracle/sj_grammar_oracle.c), each error code checked
against the unmodified reference (oracle/_ref/libsj_ref_grammar.so) before it is written.  Test infrastructure only:
run from the repository root with the reference built (make -f oracle/grammar.mk)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import grammar_oracle as G  # noqa: E402


def main():
    g, ref = G.Grammar(), G.RefGrammar()
    cases = []

    def add(doc, stream, max_depth=1024):
        s = g.stream(doc, max_depth, table=stream)
        if s is None:
            return
        r, _t, _p, starts, err, idx = s
        if stream:
            _e1, re_, rn, _n = ref.stream(doc, starts, max_depth)
            want = [G.expected_from_ref(re_[d], rn[d], starts, d, r.n) for d in range(len(starts))]
        else:
            want = [(ref.parse(doc, max_depth), None)] if r.n else [(G.EMPTY, None)]
        for d, (we, wi) in enumerate(want):
            assert G.agrees(doc, r, starts, d, int(err[d]), int(idx[d]), we, wi), (doc[:80], d, int(err[d]), int(idx[d]), we, wi)
        cases.append({"doc": doc.hex(), "stream": stream, "max_depth": max_depth, "errors": err.tolist(), "indexes": idx.tolist()})

    for doc in G.grammar_cases():
        if doc.strip():
            add(doc, False)
    for doc in G.stream_cases():
        add(doc, False)
        add(doc, True)
    for doc, md in G.depth_cases():
        if len(doc) < 5000:
            add(doc, False, md)
    cases_ = [c for c in G.grammar_cases() if c.strip()]
    add(b" ".join(cases_), True)
    with open(G.GOLDEN, "w") as f:
        json.dump({"generator": "oracle/gen_golden_document_errors.py", "cases": cases}, f, separators=(",", ":"))
    print(f"{len(cases)} cases -> {G.GOLDEN}")


if __name__ == "__main__":
    main()
