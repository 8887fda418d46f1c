"""Shared JSON parse cases: pinned renderings, edge documents and a seeded generator of valid and mutated documents."""
import json
import random

# (document member value, rendering): the simdjson path's rendering pinned in include/lc_b200.h
PINNED = [
    (b"3.14159", b"3.141590"), (b"1.23e10", b"12300000000.000000"), (b"-4.56e-3", b"-0.004560"),
    (b"-0.0", b"-0.000000"), (b"0.0078125", b"0.007812"), (b"0.0234375", b"0.023438"),
    (b"9007199254740993.0", b"9007199254740992.000000"),
    (b"9007199254740993.000000000001", b"9007199254740994.000000"),
    (b"1e308", b"%f" % 1e308), (b"1.7976931348623157e308", b"%f" % 1.7976931348623157e308),
    (b"4.9e-324", b"0.000000"), (b"2.2250738585072014e-308", b"0.000000"),
    (b"-0", b"0"), (b"0", b"0"), (b"-9223372036854775808", b"-9223372036854775808"),
    (b"-9223372036854775809", b""), (b"18446744073709551615", b"18446744073709551615"),
    (b"18446744073709551616", b""), (b"1e400", b""), (b"-1e400", b""), (b"1e-400", b"0.000000"),
    (b"-1e-400", b"-0.000000"), (b"1E2", b"100.000000"), (b"2.5e-7", b"0.000000"), (b"5e-7", b"0.000000"),
    (b"5.000001e-7", b"0.000001"), (b"1.5e-6", b"0.000002"), (b"18446744073709551615.0", b"18446744073709551616.000000"),
    (b"0.1" + b"0" * 900 + b"1", b"0.100000"), (b"123456789012345678901234567890", b""),
    (b"true", b"true"), (b"false", b"false"), (b"null", b""), (b'"a\\u0000b"', b"a\x00b"),
    (b'"\\ud83d\\ude00"', b"\xf0\x9f\x98\x80"), (b'[1, {"a" : 2}]', b'[1, {"a" : 2}]'),
]

EDGES = [b"", b"{}", b"  {}  ", b"{}\x00junk", b"{} \x00junk", b"{}x", b"[]", b"1", b'"a"', b"{", b"}",
         b'{"a":1,}', b'{"a":[1,,2]}', b'{"a":tru}', b'{"a":nul}', b'{"a":01}', b'{"a":+1}', b'{"a":1.}',
         b'{"a":.5}', b'{"a":NaN}', b'{"a":Infinity}', b'{"a":"\\ud800"}', b'{"a":"\\udc00"}', b'{"a":"\\x"}',
         b'{"a":"\x01"}', b'{"a":"\xff"}', b'{"a":"\xc0\x80"}', b'{"a":"\xed\xa0\x80"}', b'{"a":"\xf4\x90\x80\x80"}',
         b'{"a":1 "b":2}', b'{"a" 1}', b'{"a":1}}', b'{"a":{"b":[1,2,{"c":[]}]}}', b'\x00{}',
         b'{"a":1,"a":2,"content":"x"}', b'{"con\\u0074ent":"y"}', b'{"":""}', b'{"a":"\\"\\\\\\/\\b\\f\\n\\r\\t"}']


def nest(depth):
    """a root object whose member nests depth - 1 brackets (the document's depth)"""
    return b'{"a":' + b"[" * (depth - 1) + b"]" * (depth - 1) + b"}"


DEPTHS = [nest(d) for d in (2, 63, 64, 65, 66, 1024, 1025)]


def _rand_str(rng):
    out = []
    for _ in range(rng.randint(0, 12)):
        x = rng.random()
        if x < 0.6:
            out.append(chr(rng.randint(0x20, 0x7E)))
        elif x < 0.8:
            out.append(chr(rng.choice([0xE9, 0x4E2D, 0x1F600, 0x7F, 0x0, 0xA, 0x22, 0x5C])))
        else:
            out.append(chr(rng.randint(0x80, 0xFFFF)) if rng.random() < 0.5 else "\\")
    s = "".join(c for c in out if not 0xD800 <= ord(c) <= 0xDFFF)
    return s


def _rand_num(rng):
    x = rng.random()
    if x < 0.3:
        return str(rng.randint(-10 ** rng.randint(1, 21), 10 ** rng.randint(1, 21)))
    if x < 0.6:
        return "%d.%0*d" % (rng.randint(-99999, 99999), rng.randint(1, 8), rng.randint(0, 10 ** 7))
    if x < 0.8:
        return "%de%d" % (rng.randint(-999, 999), rng.randint(-330, 330))
    if x < 0.9:
        return "%d.%de%+d" % (rng.randint(0, 9), rng.randint(0, 10 ** 20), rng.randint(-30, 30))
    return repr(rng.uniform(-1e6, 1e6))


def _rand_value(rng, depth):
    x = rng.random()
    if depth < 4 and x < 0.15:
        return {_rand_str(rng): _rand_value(rng, depth + 1) for _ in range(rng.randint(0, 4))}
    if depth < 4 and x < 0.25:
        return [_rand_value(rng, depth + 1) for _ in range(rng.randint(0, 4))]
    if x < 0.55:
        return _rand_str(rng)
    if x < 0.85:
        return _Num(_rand_num(rng))
    return rng.choice([True, False, None])


class _Num(str):
    pass


def _dump(v, rng):
    ws = lambda: rng.choice(["", "", " ", "\n", "\t "])  # noqa: E731
    if isinstance(v, _Num):
        return v
    if isinstance(v, dict):
        return "{" + ",".join(ws() + json.dumps(k) + ws() + ":" + ws() + _dump(x, rng) + ws()
                              for k, x in v.items()) + "}"
    if isinstance(v, list):
        return "[" + ",".join(ws() + _dump(x, rng) + ws() for x in v) + "]"
    return json.dumps(v, ensure_ascii=rng.random() < 0.5)


def valid_docs(n, seed):
    """n valid documents with a root object (duplicate keys possible through the generator)"""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        items = [(rng.choice(["content", "a", "b", _rand_str(rng)]), _rand_value(rng, 1))
                 for _ in range(rng.randint(0, 10))]
        body = ",".join(json.dumps(k) + ":" + _dump(v, rng) for k, v in items)
        out.append(((" " if rng.random() < 0.2 else "") + "{" + body + "}").encode("utf-8", "surrogatepass"))
    return out


def mutate(docs, seed, per=4):
    """byte-level mutations of docs: deletions, insertions, replacements and truncations"""
    rng = random.Random(seed)
    alphabet = b'{}[]:,"\\ 0123456789.eE+-tfnrua\x00\x01\x7f\xc3\xa9\xed\xa0\xff'
    out = []
    for d in docs:
        for _ in range(per):
            b = bytearray(d)
            for _ in range(rng.randint(1, 3)):
                k = rng.randrange(len(b) + 1)
                x = rng.random()
                if x < 0.3 and k < len(b):
                    del b[k]
                elif x < 0.6:
                    b.insert(k, rng.choice(alphabet))
                elif x < 0.9 and k < len(b):
                    b[k] = rng.choice(alphabet)
                else:
                    b = b[:k]
            out.append(bytes(b))
    return out
