"""JSON Pointer cases shared by the oracle pinning, the host SIMT emulation and the GPU tests of sjb200_at_pointer_dev:
documents (one or a stream of several) and the pointers to look up in every one of them."""
import json
import random

import oracle_lib as O
from simdjson_b200 import corpus

# replacements of a path's last token, and tokens appended to it: a missing key, an index past the end, "-", a leading
# zero, the two escapes, a bad escape, a trailing '~', a non-digit on an array, the empty key
MUTATIONS = ["no_such_key", "999999", "18446744073709551616", "-", "01", "0", "~0", "~1", "~2", "a~", "~", "x", "", "1x", "-/0"]


def esc(k):
    return k.replace("~", "~0").replace("/", "~1")


def paths(v, depth, pre=""):
    """every pointer to a node of the parsed value v, up to `depth` tokens"""
    yield pre
    if depth == 0:
        return
    if isinstance(v, dict):
        for k, x in v.items():
            yield from paths(x, depth - 1, pre + "/" + esc(k))
    elif isinstance(v, list):
        for i, x in enumerate(v):
            yield from paths(x, depth - 1, pre + "/" + str(i))


def mutated(ps, rng, count):
    """mutations of `count` of the paths: the last token replaced, a token appended (through a scalar, or one deeper)"""
    out = []
    for p in rng.sample(ps, min(count, len(ps))):
        parent = p[: p.rfind("/")] if p else ""
        for m in MUTATIONS:
            out.append(parent + "/" + m)
            out.append(p + "/" + m)
    return out + ["", "/", "//", "x", "~", "/~01", "/statuses/-"]


def pointers_for(doc_bytes, depth, rng, nmut):
    ps = list(paths(json.loads(doc_bytes), depth))
    return ps + mutated(ps, rng, nmut)


SMALL = [
    # escaped keys: \" , é (raw and é), a surrogate pair, '/', '~', the empty key, duplicate keys
    (b'{"a\\"b":1,"\xc3\xa9":2,"\\u00e9x":3,"\\ud83d\\ude00":4,"a/b":5,"m~n":6,"":7,"d":8,"d":9,"x":{"":{"":10}}}',
     ['/a"b', "/é", "/éx", "/\U0001F600", "/a~1b", "/m~0n", "/", "/d", "/x//", "/x/", "/a/b", "/m~n", "/m~2n", "/ab"]),
    (b'[[1,2,[3,[4,5]]],{"k":[{"z":null}]},"s",true,-0.5e3,[]]',
     ["/0/2/1/1", "/0/2/1/2", "/1/k/0/z", "/1/k/0/z/q", "/1/k/-", "/5/0", "/5/-", "/2/x", "/2/~", "/4", "/6", "/00", "/0/-/1", "/1/k/0/", "/3/~2"]),
    (b'"root string"', ["", "/", "/a", "/~", "/~x", "x"]),
    (b'12345', ["", "/0", "/~1", "/~q/~1"]),
    (b'{}', ["", "/", "/a", "~"]),
    (b'[]', ["", "/0", "/-", "/", "/a", "/01"]),
]

# documents with a bad number or atom: every pointer answers the first token in error
BAD = [b'{"a":[1,2,tru],"b":1}', b'[1,2,-,{"a":3}]', b'{"a":"x","b":01}', b'{"a":nul}', b'[1.5e,2]', b'{"a":[1,2,3],"b":fals}']


def stream_of(rows):
    """NDJSON of the rows, and the structural index at which each row starts"""
    return b"\n".join(rows) + b"\n"


def random_docs(n, seed):
    rng = random.Random(seed)
    return [bytes(corpus.random_json(rng.randrange(100, 4000), seed=seed * 1000 + i)) for i in range(n)]


def twitter_rows():
    """the statuses of twitter.json as NDJSON object rows"""
    t = json.loads(O.jsonexample("twitter.json"))
    return [json.dumps(s, ensure_ascii=False).encode() for s in t["statuses"]]


def amazon_rows(k=200):
    return O.jsonexample("amazon_cellphones.ndjson").split(b"\n")[:k]


def corpus_cases(full=True):
    """[(name, document bytes, pointers)]: twitter (every path up to depth 4 when full, else 3), citm, the small and bad
    documents, seeded random documents from corpus.py"""
    rng = random.Random(0x9017)
    tw = O.jsonexample("twitter.json")
    citm = O.jsonexample("citm_catalog.json")
    out = [("twitter.json", tw, pointers_for(tw, 4 if full else 3, rng, 300 if full else 60)),
           ("citm_catalog.json", citm, pointers_for(citm, 3 if full else 2, rng, 100 if full else 30))]
    out += [(f"small{i}", d, ps) for i, (d, ps) in enumerate(SMALL)]
    out += [(f"bad{i}", d, ["", "/a", "/0", "/b", "/3/a"]) for i, d in enumerate(BAD)]
    for i, d in enumerate(random_docs(8 if full else 4, 7)):
        out.append((f"random{i}", d, pointers_for(d, 3, rng, 20)))
    return out
