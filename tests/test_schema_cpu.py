"""CPU: the JSON schema `format` (gl_format_schema): the compiler and the automaton of the schema mask kernel, compiled for the
host through tests/hostcheck/schema_shim.cpp, against the restatement in tests/schema_oracle.py and against jsonschema's
Draft 2020-12 validator; the refusals; the ABI; the service with json_schema=True over an engine double."""
import asyncio
import ctypes
import json
import os
import random
import subprocess

import numpy as np
import pytest

import json_oracle as J
import schema_oracle as SO
from conftest import ROOT

# ---- the schemas ---------------------------------------------------------------------------------------------------------
# pydantic 2.13 model_json_schema() output, as literals:
#   class Address(BaseModel): street: str; city: str; zip: Optional[str] = None
#   class Person(BaseModel): name: str; age: int; email: Optional[str] = None; addresses: List[Address] = []; tags: List[str]
PYD_PERSON = {"$defs": {"Address": {"properties": {"street": {"title": "Street", "type": "string"}, "city": {"title": "City", "type": "string"},
                                                   "zip": {"anyOf": [{"type": "string"}, {"type": "null"}], "default": None, "title": "Zip"}},
                                    "required": ["street", "city"], "title": "Address", "type": "object"}},
              "properties": {"name": {"title": "Name", "type": "string"}, "age": {"title": "Age", "type": "integer"},
                             "email": {"anyOf": [{"type": "string"}, {"type": "null"}], "default": None, "title": "Email"},
                             "addresses": {"default": [], "items": {"$ref": "#/$defs/Address"}, "title": "Addresses", "type": "array"},
                             "tags": {"items": {"type": "string"}, "title": "Tags", "type": "array"}},
              "required": ["name", "age", "tags"], "title": "Person", "type": "object"}
#   class Color(str, Enum): red = "red"; green = "green"
#   class Item(BaseModel): color: Color; count: int = 1; ok: bool
PYD_ENUM = {"$defs": {"Color": {"enum": ["red", "green"], "title": "Color", "type": "string"}},
            "properties": {"color": {"$ref": "#/$defs/Color"}, "count": {"default": 1, "title": "Count", "type": "integer"},
                           "ok": {"title": "Ok", "type": "boolean"}},
            "required": ["color", "ok"], "title": "Item", "type": "object"}
#   class Tree(BaseModel): value: int; children: List["Tree"] = []
PYD_TREE = {"$defs": {"Tree": {"properties": {"value": {"title": "Value", "type": "integer"},
                                              "children": {"default": [], "items": {"$ref": "#/$defs/Tree"}, "title": "Children", "type": "array"}},
                               "required": ["value"], "title": "Tree", "type": "object"}},
            "$ref": "#/$defs/Tree"}
#   class Leaf(BaseModel): kind: Literal["leaf"]; note: Optional[str] = None
#   class Wrap(BaseModel): leaf: Leaf; score: float; maybe: Optional[int] = None
PYD_NESTED = {"$defs": {"Leaf": {"properties": {"kind": {"const": "leaf", "title": "Kind", "type": "string"},
                                                "note": {"anyOf": [{"type": "string"}, {"type": "null"}], "default": None, "title": "Note"}},
                                 "required": ["kind"], "title": "Leaf", "type": "object"}},
              "properties": {"leaf": {"$ref": "#/$defs/Leaf"}, "score": {"title": "Score", "type": "number"},
                             "maybe": {"anyOf": [{"type": "integer"}, {"type": "null"}], "default": None, "title": "Maybe"}},
              "required": ["leaf", "score"], "title": "Wrap", "type": "object"}

SCHEMAS = [
    {"type": "object"},
    {"type": "object", "properties": {}},
    {"type": "object", "properties": {"name": {"type": "string"}, "age": {"type": "integer"}}, "required": ["name", "age"]},
    {"type": "object", "properties": {"a": {"type": "string"}, "b": {"type": "integer"}, "c": {"type": "boolean"}}},
    {"type": "object", "properties": {"a": {"type": "integer"}, "b": {"type": "number"}}, "required": ["b"]},
    {"type": "object", "properties": {"s": {"type": "string", "minLength": 2, "maxLength": 4}}, "required": ["s"]},
    {"type": "object", "properties": {"xs": {"type": "array", "items": {"type": "integer"}, "minItems": 1, "maxItems": 3}}, "required": ["xs"]},
    {"type": "object", "properties": {"xs": {"type": "array"}}, "required": ["xs"]},
    {"type": "object", "properties": {"e": {"enum": ["a", "ab", 4, 42, -1, True, None]}}, "required": ["e"]},
    {"type": "object", "properties": {"c": {"const": "fixed"}, "n": {"const": 0}}, "required": ["c", "n"]},
    {"type": "object", "properties": {"v": {"type": ["string", "null"]}}, "required": ["v"]},
    {"type": "object", "properties": {"v": {"anyOf": [{"type": "string", "maxLength": 3}, {"type": "integer"}, {"type": "null"}]}}, "required": ["v"]},
    {"type": "object", "properties": {"v": {"oneOf": [{"type": "boolean"}, {"type": "array", "items": {"type": "string"}}]}}},
    {"type": "object", "properties": {"o": {"type": "object"}}, "required": ["o"]},
    {"type": "object", "properties": {"o": {"type": "object", "properties": {"k": {"type": "null"}}, "additionalProperties": False}}, "required": ["o"]},
    {"type": "object", "properties": {"q\"u\\o\nte": {"type": "string"}, "café ✓": {"enum": ["é", "tab\there", "\u0001"]}}, "required": ["café ✓"]},
    {"type": "object", "properties": {"x": {"allOf": [{"type": "integer"}]}, "y": True, "z": {}}, "required": ["x"]},
    {"properties": {"x": {"type": "number"}}, "required": ["x"], "title": "T", "description": "d", "$schema": "https://json-schema.org/draft/2020-12/schema"},
    {"type": "object", "properties": {"self": {"$ref": "#"}}},
    {"definitions": {"P": {"type": "object", "properties": {"p": {"type": "integer"}}, "required": ["p"]}},
     "type": "object", "properties": {"a": {"$ref": "#/definitions/P"}, "b": {"items": {"$ref": "#/definitions/P"}, "maxItems": 2}}, "required": ["a"]},
    {"type": "object", "properties": {"n": {"type": ["integer", "number"]}, "t": {"type": ["boolean", "string", "null"], "maxLength": 1}}},
    {"type": "object", "properties": {"deep": {"type": "array", "items": {"type": "array", "items": {"type": "array", "items": {"type": "integer"}}}}}},
    {"type": "object", "properties": {"a": {"type": "string", "minLength": 1}, "b": {"type": "string", "maxLength": 0}}, "required": ["a", "b"]},
    {"type": "object", "properties": {"arr": {"type": "array", "items": {"enum": [1, 2, 3]}, "minItems": 2, "maxItems": 2}}, "required": ["arr"]},
    {"type": "object", "properties": {"k1": {"type": "integer"}, "k10": {"type": "integer"}, "k2": {"type": "integer"}}, "required": ["k10"]},
    PYD_PERSON,
    PYD_ENUM,
    PYD_TREE,
    PYD_NESTED,
    {"$defs": {"L": {"type": "object", "properties": {"next": {"anyOf": [{"$ref": "#/$defs/L"}, {"type": "null"}]}, "v": {"type": "integer"}}, "required": ["v", "next"]}},
     "$ref": "#/$defs/L"},
]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """CPU build of schema_compile.cpp + schema_fsm.h through tests/hostcheck/schema_shim.cpp -- test infrastructure only"""
    out = str(tmp_path_factory.mktemp("schemafsm") / "libschemafsm.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "schema_shim.cpp"),
                           os.path.join(ROOT, "gridllm_b200", "csrc", "schema_compile.cpp")])
    L = ctypes.CDLL(out)
    L.sf_error.restype = ctypes.c_char_p
    L.sf_compile.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.sf_run.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.sf_allowed.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                             ctypes.c_char_p]
    assert L.sf_state_bytes() == 280
    return L


def _text(schema):
    return json.dumps(schema, ensure_ascii=False, separators=(",", ":")).encode("utf-8")


def compile_c(L, schema):
    """-> (code, blob or message)"""
    raw = schema if isinstance(schema, bytes) else _text(schema)
    buf = ctypes.create_string_buffer(1 << 20)
    n = ctypes.c_int(0)
    rc = L.sf_compile(raw, len(raw), buf, len(buf), ctypes.byref(n))
    return (rc, buf.raw[: n.value]) if rc == 0 else (rc, L.sf_error().decode())


def c_run(L, blob, data):
    done = ctypes.c_int(0)
    n = L.sf_run(blob, bytes(data), len(data), ctypes.byref(done))
    return n == len(data), n == len(data) and bool(done.value)


ALPHABET = [bytes([b]) for b in list(range(0x20, 0x7F)) + [0x09, 0x0A] + list(range(0x80, 0xC0)) + [0xC3, 0xE2, 0xF0]]


def c_allowed(L, blob, prefix, pieces=ALPHABET):
    offs = np.zeros(len(pieces) + 1, np.int32)
    offs[1:] = np.cumsum([len(p) for p in pieces])
    out = ctypes.create_string_buffer(len(pieces))
    done = L.sf_allowed(blob, bytes(prefix), len(prefix), b"".join(pieces), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), len(pieces), out)
    assert done >= 0, prefix
    return [bool(x) for x in out.raw], bool(done)


# ---- conforming documents ------------------------------------------------------------------------------------------------
def _ws(rnd):
    return rnd.choice(["", "", " ", "\n", "\n  ", "\n\t"])


def _gen(rnd, n, d, budget):
    """a document of oracle node n (text), key order required-first, random optional subsets and ws"""
    if n.kind == "union":
        n = rnd.choice([a for a in n.alts if d + a.mind <= SO.MAX_DEPTH and (a.mind < 2 or budget > 0)] or n.alts[:1])
    k = n.kind
    if k in ("any", "objany"):
        return rnd.choice(["{}", '{"k": [1, "x"]}'] if k == "objany" else ["1", '"s"', "null", "[true, {}]", "{}"])
    if k == "str":
        hi = min(n.hi, n.lo + 4)
        return json.dumps("".join(rnd.choice("ab é\"\\\n✓") for _ in range(rnd.randint(n.lo, hi))), ensure_ascii=rnd.random() < 0.3)
    if k == "int":
        return str(rnd.randint(-500, 500))
    if k == "num":
        return rnd.choice(["0", "-1.5", "3e8", "2.25E-3", "17"])
    if k == "bool":
        return rnd.choice(["true", "false"])
    if k == "null":
        return "null"
    if k == "enum":
        return rnd.choice(n.lits).decode("utf-8")
    if k == "arr":
        cnt = rnd.randint(n.lo, min(n.hi, n.lo + (3 if budget > 0 else 0)))
        items = [_gen(rnd, n.items, d + 1, budget - 1) for _ in range(cnt)]
        return "[" + _ws(rnd) + ("," + _ws(rnd)).join(i + _ws(rnd) for i in items) + "]"
    keys = list(range(n.nreq)) + [j for j in range(n.nreq, len(n.props)) if budget > 0 and rnd.random() < 0.5]
    parts = [n.props[j][0].decode("utf-8") for j in keys]
    body = ("," + _ws(rnd)).join('"' + p + _ws(rnd) + ":" + _ws(rnd) + _gen(rnd, n.props[j][1], d + 1, budget - 1) + _ws(rnd)
                                  for p, j in zip(parts, keys))
    return "{" + _ws(rnd) + body + "}"


def documents(schema, seed, n=25):
    rnd = random.Random(seed)
    root = SO.compile_schema(schema)
    return [(_gen(rnd, root, 0, 3) + rnd.choice(["", " ", "\n"])).encode("utf-8") for _ in range(n)]


def _mutate(rnd, doc):
    b = bytearray(doc)
    for _ in range(rnd.randint(1, 3)):
        op = rnd.randrange(3)
        i = rnd.randrange(len(b) + 1)
        if op == 0 and b:
            del b[min(i, len(b) - 1)]
        elif op == 1:
            b.insert(i, rnd.choice(b'{}[]",:0123456789-.eE tfn\\a\n'))
        elif b:
            b[min(i, len(b) - 1)] = rnd.choice(b'{}[]",: 1aZ')
    return bytes(b)


# ---- tests -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(SCHEMAS)))
def test_completeness_and_agreement_on_every_prefix(lib, i):
    import jsonschema
    schema = SCHEMAS[i]
    rc, blob = compile_c(lib, schema)
    assert rc == 0, blob
    root = SO.compile_schema(schema)
    val = jsonschema.Draft202012Validator(schema)
    rnd = random.Random(100 + i)
    docs = documents(schema, seed=i)
    for doc in docs:
        assert val.is_valid(json.loads(doc)), doc                  # the generator writes documents of the schema
        assert c_run(lib, blob, doc) == (True, True), doc          # completeness: accepted whole
        assert SO.run(root, doc) == (True, True), doc
    inputs = docs + [_mutate(rnd, rnd.choice(docs)) for _ in range(150)]
    for data in inputs:
        for k in range(len(data) + 1):
            assert c_run(lib, blob, data[:k]) == SO.run(root, data[:k]), (data[:k], schema)


def _walk(L, blob, rnd, max_len=400):
    """a random walk of the automaton over single bytes and a few multi-byte pieces, biased to close"""
    out = b""
    closers = set(b'}]"')
    for _ in range(max_len):
        allowed, done = c_allowed(L, blob, out)
        opts = [ALPHABET[j] for j, a in enumerate(allowed) if a]
        assert opts or done, out                                # no dead ends
        if done and (not opts or rnd.random() < 0.5):
            return out, True
        close = [p for p in opts if p[0] in closers or p in (b"0", b"1", b"n", b"t")]
        pick = rnd.choice(close) if close and rnd.random() < 0.6 else rnd.choice(opts)
        out += pick
    return out, False


def _close(L, blob, out, limit=3000):
    """from any reached state a closing walk finishes a document: prefer closers, short literals, no ws"""
    rank = {c: i for i, c in enumerate(b'"}],:0123456789ntf{[a')}
    for _ in range(limit):
        allowed, done = c_allowed(L, blob, out)
        if done:
            return out
        opts = [ALPHABET[j] for j, a in enumerate(allowed) if a]
        assert opts, out
        out += min(opts, key=lambda p: rank.get(p[0], 99))
    raise AssertionError(("no close", out[-80:]))


@pytest.mark.parametrize("i", range(len(SCHEMAS)))
def test_random_walks_are_sound_and_never_dead_end(lib, i):
    import jsonschema
    schema = SCHEMAS[i]
    rc, blob = compile_c(lib, schema)
    assert rc == 0, blob
    root = SO.compile_schema(schema)
    val = jsonschema.Draft202012Validator(schema)
    rnd = random.Random(7 + i)
    for w in range(40):
        out, done = _walk(lib, blob, rnd, max_len=rnd.choice([30, 120, 400]))
        if not done:
            out = _close(lib, blob, out)
        assert SO.run(root, out) == (True, True), out
        assert val.is_valid(json.loads(out)), (out, schema)
        if w % 8 == 0:                                           # the automaton's mask equals the oracle's at a few cuts
            for k in sorted(rnd.sample(range(len(out) + 1), min(4, len(out) + 1))):
                allowed, _ = c_allowed(lib, blob, out[:k])
                assert allowed == [SO.viable(root, out[:k] + p) for p in ALPHABET], (out[:k], schema)


def test_recursive_required_ref_never_dead_ends(lib):
    # a required recursive property: refused outright (no finite document)
    rc, msg = compile_c(lib, {"$defs": {"N": {"type": "object", "properties": {"n": {"$ref": "#/$defs/N"}}, "required": ["n"]}}, "$ref": "#/$defs/N"})
    assert rc == -4 and "deeper than 64" in msg
    # an optional recursive one: at depth 63 the key can no longer be taken; the walk still closes
    rc, blob = compile_c(lib, {"type": "object", "properties": {"n": {"$ref": "#"}, "xs": {"type": "array", "items": {"$ref": "#"}, "minItems": 1}}})
    assert rc == 0
    deep = b'{"n":' * 63
    allowed, _ = c_allowed(lib, blob, deep)
    assert allowed[ALPHABET.index(b"{")]
    allowed, _ = c_allowed(lib, blob, deep + b"{")
    assert not allowed[ALPHABET.index(b'"')] and allowed[ALPHABET.index(b"}")]         # depth 64: no key fits
    out = _close(lib, blob, deep + b"{")
    assert json.loads(out) is not None


REFUSALS = [
    ({"type": "object", "properties": {"zip": {"type": "string", "pattern": "^[0-9]+$"}}}, -4, "'pattern' is not supported at /properties/zip"),
    ({"type": "object", "properties": {"d": {"type": "string", "format": "date"}}}, -4, "'format' is not supported at /properties/d"),
    ({"type": "object", "properties": {"n": {"type": "integer", "minimum": 0}}}, -4, "'minimum' is not supported at /properties/n"),
    ({"type": "object", "properties": {"n": {"type": "number", "exclusiveMaximum": 3}}}, -4, "'exclusiveMaximum' is not supported at /properties/n"),
    ({"type": "object", "properties": {"n": {"type": "number", "multipleOf": 3}}}, -4, "'multipleOf' is not supported at /properties/n"),
    ({"type": "object", "properties": {"a": {"type": "array", "uniqueItems": True}}}, -4, "'uniqueItems' is not supported at /properties/a"),
    ({"type": "object", "properties": {"a": {"prefixItems": [{"type": "string"}]}}}, -4, "'prefixItems' is not supported at /properties/a"),
    ({"type": "object", "patternProperties": {"x": {}}}, -4, "'patternProperties' is not supported at /"),
    ({"type": "object", "properties": {"a": {"not": {"type": "null"}}}}, -4, "'not' is not supported at /properties/a"),
    ({"type": "object", "if": {}, "then": {}}, -4, "'if' is not supported at /"),
    ({"type": "object", "additionalProperties": True}, -4, "'additionalProperties' other than false is not supported at /additionalProperties"),
    ({"type": "object", "properties": {"a": {}}, "additionalProperties": {"type": "string"}}, -4, "at /additionalProperties"),
    ({"type": "object", "properties": {"a": {}}, "required": ["b"]}, -4, "required property 'b' is not in 'properties' at /required"),
    ({"type": "array"}, -4, "the root must be an object schema"),
    ({"type": "object", "properties": {"e": {"enum": []}}}, -4, "empty 'enum' (no document) at /properties/e"),
    ({"type": "object", "properties": {"e": {"enum": [1.5]}}}, -4, "at /properties/e"),
    ({"type": "object", "properties": {"s": {"type": "string", "minLength": 3, "maxLength": 2}}}, -4, "'minLength' > 'maxLength' (no document) at /properties/s"),
    ({"type": "object", "properties": {"a": {"type": "array", "minItems": 3, "maxItems": 1}}}, -4, "'minItems' > 'maxItems' (no document) at /properties/a"),
    ({"type": "object", "properties": {"s": {"type": "string", "maxLength": 70000}}}, -4, "'maxLength' above 65534 at /properties/s"),
    ({"type": "object", "properties": {"v": {"anyOf": [{"type": "integer"}, {"type": "number"}]}}}, -4, "same byte ('-') are not supported at /properties/v"),
    ({"type": "object", "properties": {"v": {"anyOf": [{"type": "string"}, {"enum": ["x"]}]}}}, -4, "at /properties/v"),
    ({"type": "object", "properties": {"v": {"allOf": [{"type": "string"}, {"maxLength": 2}]}}}, -4, "'allOf' with other than one member is not supported at /properties/v"),
    ({"type": "object", "properties": {"v": {"$ref": "https://example.com/s.json"}}}, -4, "is not a local reference at /properties/v"),
    ({"type": "object", "properties": {"v": {"$ref": "#/$defs/missing"}}}, -4, "at /properties/v"),
    ({"type": "object", "properties": {"p%d" % i: {"type": "integer"} for i in range(256)}}, -4, "more than 255 properties at /"),
    ({"$defs": {"A": {"$ref": "#/$defs/B"}, "B": {"$ref": "#/$defs/A"}}, "type": "object", "properties": {"a": {"$ref": "#/$defs/A"}}}, -4, "cycle"),
    ({"type": "object", "properties": {"a": False}}, -4, "at /properties/a"),
    ({"type": "object", "properties": {"a~/b": {"type": "string", "pattern": "x"}}}, -4, "at /properties/a~0~1b"),
    (b'{"type": "object",', -1, "malformed JSON"),
    (b'{"type": "object", "type": "object"}', -1, "duplicate key"),
    (b'[1, 2', -1, "malformed JSON"),
    ({"type": "object", "properties": {"s": {"type": "string", "minLength": -1}}}, -1, "'minLength' must be a non-negative integer"),
    ({"type": "object", "properties": {"s": {"type": "strng"}}}, -1, "unknown type 'strng' at /properties/s"),
]


@pytest.mark.parametrize("i", range(len(REFUSALS)))
def test_refusals_name_the_keyword_and_pointer(lib, i):
    schema, code, text = REFUSALS[i]
    rc, msg = compile_c(lib, schema)
    assert rc == code and text in msg, (rc, msg)


def test_node_limit(lib):
    props = {"p%d" % i: {"type": "object", "properties": {"q%d" % j: {"type": "integer"} for j in range(20)}} for i in range(200)}
    rc, msg = compile_c(lib, {"type": "object", "properties": props})
    assert rc == -4 and "4096 nodes" in msg


def test_canonical_literals(lib):
    """keys and enum members only in Python's json.dumps(ensure_ascii=False) spelling"""
    schema = {"type": "object", "properties": {"é\n": {"enum": ["\u0007é", 10]}}, "required": ["é\n"]}
    rc, blob = compile_c(lib, schema)
    assert c_run(lib, blob, '{"é\\n":"\\u0007é"}'.encode()) == (True, True)
    assert c_run(lib, blob, b'{"\\u00e9\\n":')[0] is False                 # an escaped spelling of the key
    assert c_run(lib, blob, '{"é\\n":"\\u0007\\u00e9"}'.encode())[0] is False
    assert c_run(lib, blob, '{"é\\n":"\\u0007é"'.encode()) == (True, False)
    assert c_run(lib, blob, '{"é\\n":10}'.encode()) == (True, True)
    assert c_run(lib, blob, '{"é\\n":1}'.encode())[0] is False
    assert c_run(lib, blob, '{"é\\n":10.0}'.encode())[0] is False


def test_key_order_and_subsets(lib):
    schema = {"type": "object", "properties": {"a": {"type": "integer"}, "b": {"type": "integer"}, "c": {"type": "integer"}}, "required": ["c"]}
    rc, blob = compile_c(lib, schema)
    assert c_run(lib, blob, b'{"c":1,"a":2,"b":3}') == (True, True)
    assert c_run(lib, blob, b'{"c":1,"b":3}') == (True, True)
    assert c_run(lib, blob, b'{"c":1}') == (True, True)
    assert not c_run(lib, blob, b'{"a":2')[0]                   # the required key first
    assert not c_run(lib, blob, b'{"c":1,"b":3,"a"')[0]         # optional ones in properties order
    assert not c_run(lib, blob, b'{"c":1,"c"')[0]
    assert not c_run(lib, blob, b'{}')[0]


# ---- ABI -------------------------------------------------------------------------------------------------------------------
def test_abi():
    from gridllm_b200 import native as N
    assert ctypes.sizeof(N.SampleOpts) == 72 and N.SampleOpts.format.offset == 64
    assert "gl_format_schema" in N.ABI_SYMBOLS and N.GL_FORMAT_SCHEMA_BASE == 256
    hdr = open(os.path.join(ROOT, "include", "gridllm_native.h")).read()
    assert "#define GL_ABI_VERSION 2" in hdr and "#define GL_FORMAT_SCHEMA_BASE 256" in hdr
    assert "int  gl_format_schema(gl_engine* e, const char* schema_utf8, int32_t n_bytes, int32_t* format_out);" in hdr
    import re
    declared = set(re.findall(r"\b(gl_[a-z_]+)\s*\(", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)))
    assert declared == set(N.ABI_SYMBOLS)


# ---- the service with json_schema=True ---------------------------------------------------------------------------------------
def _schema_double():
    from test_json_cpu import _json_double
    base = _json_double()

    class SchemaDouble(base):
        """the JSON double with schemas: a dict format (or a registered code) draws through the schema oracle's mask"""
        def format_schema(self, schema):
            from gridllm_b200 import native as N
            if not hasattr(self, "_lib_s"):
                self._lib_s, self._codes, self._roots = _LIB[0], {}, {}
            text = _text(schema)
            rc, blob = compile_c(self._lib_s, text)
            if rc != 0:
                raise N.NativeError(rc, blob)
            if text not in self._codes:
                self._codes[text] = 256 + len(self._codes)
                self._roots[self._codes[text]] = SO.compile_schema(json.loads(text))
            return self._codes[text]

        def _draw(self, logits, gen, stops, opts, i, fmt):
            from oracle import sampler as SM
            if isinstance(fmt, dict):
                root = self._roots[self.format_schema(fmt)]
                pieces = self._pieces()
                logits = SO.apply_mask(root, logits + self.bias * self._bonus, pieces, stops, gen)
                return SM.sample(logits, *opts, i)
            return super()._draw(logits, gen, stops, opts, i, fmt)

    return SchemaDouble


_LIB = []


def _run(coro):
    return asyncio.new_event_loop().run_until_complete(coro)


@pytest.mark.parametrize("max_batch", [0, 4])
def test_service_enforces_schemas(lib, tiny_gguf, hostcheck_lib, monkeypatch, max_batch):
    import jsonschema
    import oracle_engine
    from gridllm_b200 import service as SV
    _LIB[:] = [lib]
    oracle_engine.use_hostcheck(hostcheck_lib)
    Double = _schema_double()
    monkeypatch.setattr(SV.N, "Engine", Double)
    monkeypatch.setattr(SV.N, "device_count", lambda: 1)
    schema = {"type": "object", "properties": {"ok": {"type": "boolean"}, "n": {"enum": [1, 2]}}, "required": ["ok", "n"]}
    svc = SV.NativeInferenceService({"tiny:latest": tiny_gguf}, device=0, max_batch=max_batch, json_schema=True)
    try:
        eng = svc._engine("tiny:latest")
        Double.bias = 50.0
        req = {"id": "s1", "model": "tiny:latest", "prompt": "give me json", "priority": "medium",
               "options": {"num_predict": 40, "temperature": 0}, "metadata": {"format": schema}}
        res = _run(svc.generateResponse(req))
        assert eng.formats[-1] == schema and res["done_reason"] == "stop"
        jsonschema.validate(json.loads(res["response"]), schema)

        async def collect(r):
            return [c async for c in svc.generateStreamResponse(r)]
        text = "".join(c["response"] for c in _run(collect(dict(req, id="s2"))))
        assert text == res["response"]
        chat = {"id": "c1", "model": "tiny:latest", "priority": "low", "options": {"num_predict": 40, "format": schema},
                "metadata": {"messages": [{"role": "user", "content": "json please"}]}}
        out = _run(svc.generateChatResponse(chat))
        jsonschema.validate(json.loads(out["message"]["content"]), schema)
        # "json" still means the plain JSON mask
        out = _run(svc.generateResponse(dict(req, id="s3", metadata={"format": "json"})))
        assert eng.formats[-1] == "json" and isinstance(json.loads(out["response"]), dict)
        # a schema outside the subset fails the request before it runs
        bad = {"type": "object", "properties": {"zip": {"type": "string", "pattern": "^[0-9]{5}$"}}}
        n_before = len(eng.formats)
        with pytest.raises(RuntimeError) as ei:
            _run(svc.generateResponse(dict(req, id="s4", metadata={"format": bad})))
        assert str(ei.value) == "Inference failed: format schema: 'pattern' is not supported at /properties/zip"
        assert len(eng.formats) == n_before
    finally:
        Double.bias = 0.0
        svc.close()
