"""Typed-column cases shared by the oracle pinning, the host SIMT emulation and the GPU tests of sjb200_column_dev:
documents and the pointers whose results feed every getter."""
import json

import pointer_cases as PC

# integer edges, floats, atoms: INT64_MIN, INT64_MAX, INT64_MAX + 1, UINT64_MAX, -1, 0, -0, 1.5, true, false, null
EDGES = (b'{"min":-9223372036854775808,"max":9223372036854775807,"over":9223372036854775808,"umax":18446744073709551615,'
         b'"m1":-1,"zero":0,"nzero":-0,"half":1.5,"exp":-2.5e-3,"t":true,"f":false,"n":null,"s":"1","a":[1],"o":{"k":1}}')
EDGE_POINTERS = ["/min", "/max", "/over", "/umax", "/m1", "/zero", "/nzero", "/half", "/exp", "/t", "/f", "/n", "/s", "/a", "/a/0", "/o", "/o/k",
                 "", "/missing", "/a/1"]

# 1e400: the reference's parse fails (NUMBER_ERROR: the value is infinite); the tokens only check float grammar, so on the
# device the row is a 'd' value, INCORRECT_TYPE under every kind but the float getter (not on the device)
INFINITE = b'{"big":1e400,"x":1}'

# strings: empty, escapes, \u0000 inside, a surrogate pair, and lengths 1-33 around the 16-byte vector width
STRINGS = json.dumps(["", 'a"b\\\n\t/', "x\u0000y\u0000", "\U0001F600é", "€" * 7] + ["abcdefghijklmnopqrstuvwxyz0123456789"[:k] for k in range(1, 34)],
                     ensure_ascii=False).encode()
STRING_POINTERS = [f"/{i}" for i in range(38)] + ["/38", ""]

# containers: empty ones, duplicate keys, nesting, keys whose values are strings (a string at depth 0 not followed by ':')
CONTAINERS = (b'{"e":[],"o":{},"d":{"k":1,"k":2,"k":"v","k":{}},"n":[[1,2],{"a":[]},[],"s",null],"sv":{"a":"b","c":"d"},'
              b'"deep":[[[[[1]]]],[[]],{"x":{"y":[1,2,3]}}]}')
CONTAINER_POINTERS = ["", "/e", "/o", "/d", "/n", "/n/0", "/n/1", "/n/1/a", "/n/2", "/n/3", "/sv", "/deep", "/deep/0", "/deep/2/x/y", "/d/k", "/zz"]


def long_containers():
    """an array and an object longer than the warp walk's 4 096 structurals and than one CTA step"""
    arr = json.dumps([{"i": i, "v": [i, str(i)]} if i % 3 else [i, [i]] for i in range(3000)]).encode()
    obj = json.dumps({f"k{i}": ([i] * (i % 4) if i % 2 else {"x": i, "y": [1, {}]}) for i in range(5000)}).encode()
    return [(arr, ["", "/0", "/1", "/2999", "/1500/v"]), (obj, ["", "/k0", "/k1", "/k4999", "/k3"])]


def big_array(n=16777216):
    """an array of n elements (16 777 216: one past the tape count's 0xFFFFFF)"""
    return b"[" + b"0," * (n - 1) + b"0]"


TWITTER_POINTERS = ["/id", "/user/id", "/user/screen_name", "/text", "/favorited", "/entities/hashtags", "/user", "/retweeted_status/id"]


def documents():
    """[(name, document, pointers)]: single documents, each parsed by the reference as a whole"""
    out = [("edges", EDGES, EDGE_POINTERS), ("strings", STRINGS, STRING_POINTERS), ("containers", CONTAINERS, CONTAINER_POINTERS)]
    out += [(f"small{i}", d, ps) for i, (d, ps) in enumerate(PC.SMALL)]
    out += [(f"bad{i}", d, ["", "/a", "/0", "/b"]) for i, d in enumerate(PC.BAD)]
    out += [(f"row{i}", r, TWITTER_POINTERS) for i, r in enumerate(PC.twitter_rows()[:12])]
    out += [(f"long{i}", d, ps) for i, (d, ps) in enumerate(long_containers())]
    return out


def document(name):
    """the document of documents() called name"""
    return {n: d for n, d, _p in documents()}[name]
