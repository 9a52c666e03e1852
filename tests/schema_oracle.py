"""TEST INFRASTRUCTURE: the language of a JSON schema `format` (include/gridllm_native.h, gl_format_schema) restated in Python,
and the mask it implies over a vocabulary.

The restatement is a recursive-descent parser written as Python generators (one per value being read, fed one byte at a time),
written independently of the flat automaton of gridllm_b200/csrc/schema_fsm.h.  The lexical rules of the JSON language
(string bodies, number syntax) come from tests/json_oracle.py; the ws rule, the nesting bound and every schema rule are
restated here:
  - objects with properties: the required keys in `properties` order, then any subset of the optional ones in that order;
  - keys and enum members in canonical spelling (json.dumps(x, ensure_ascii=False));
  - strings count code points, an escape counting as one; integers have no fraction or exponent;
  - anyOf / oneOf / type lists pick the alternative by the first byte;
  - no dead ends: a value whose smallest document cannot close within depth 64 is never started, an optional key whose value
    cannot is never taken, and ',' only where another key or item can follow."""
import json

import json_oracle as J

MAX_DEPTH = 64
INF = 10 ** 6


class Reject(Exception):
    pass


class Node:
    def __init__(self, kind, **kw):
        self.kind = kind
        self.__dict__.update(kw)
        self.mind = INF


def canon(x):
    return json.dumps(x, ensure_ascii=False).encode("utf-8")


def compile_schema(schema):
    """schema (a dict) -> root Node; the schema is assumed to lie inside the subset"""
    memo = {}

    def ref(r):
        if r == "#":
            return schema
        for pre, key in (("#/$defs/", "$defs"), ("#/definitions/", "definitions")):
            if r.startswith(pre):
                return schema[key][r[len(pre):].replace("~1", "/").replace("~0", "~")]
        raise ValueError(r)

    def node(s):
        if s is True:
            s = {}
        if id(s) in memo:
            return memo[id(s)]
        if "$ref" in s:
            memo[id(s)] = n = node(ref(s["$ref"]))
            return n
        if "allOf" in s:
            memo[id(s)] = n = node(s["allOf"][0])
            return n
        alts = s.get("anyOf", s.get("oneOf"))
        if alts is not None:
            u = memo[id(s)] = Node("union", alts=[])
            u.alts = [node(a) for a in alts]
            return u
        types = s.get("type")
        types = [types] if isinstance(types, str) else list(types or [])
        if "enum" in s or "const" in s:
            members = s["enum"] if "enum" in s else [s["const"]]
            ok = lambda m: not types or any(
                t == {str: "string", bool: "boolean", type(None): "null", int: "integer"}[type(m)] or (t == "number" and type(m) is int)
                for t in types)
            lits = []
            for m in members:
                if ok(m) and canon(m) not in lits:
                    lits.append(canon(m))
            memo[id(s)] = n = Node("enum", lits=lits)
            return n
        if not types:
            if {"properties", "required", "additionalProperties"} & s.keys():
                types = ["object"]
            elif {"items", "minItems", "maxItems"} & s.keys():
                types = ["array"]
            elif {"minLength", "maxLength"} & s.keys():
                types = ["string"]
            else:
                memo[id(s)] = n = Node("any")
                return n
        if "number" in types:
            types = [t for t in types if t != "integer"]
        types = list(dict.fromkeys(types))
        u = None
        if len(types) > 1:
            u = memo[id(s)] = Node("union", alts=[])
        out = []
        for t in types:
            if t == "object":
                if "properties" not in s and "additionalProperties" not in s:
                    n = Node("objany")
                else:
                    props = s.get("properties", {})
                    req = [k for k in props if k in s.get("required", [])]
                    n = Node("obj", props=[], nreq=len(req))
                    if u is None:
                        memo[id(s)] = n
                    order = req + [k for k in props if k not in req]
                    n.props = [(canon(k)[1:], node(props[k])) for k in order]
            elif t == "array":
                n = Node("arr", lo=s.get("minItems", 0), hi=s.get("maxItems", INF), items=None)
                if u is None:
                    memo[id(s)] = n
                n.items = node(s["items"]) if "items" in s else Node("any")
            elif t == "string":
                n = Node("str", lo=s.get("minLength", 0), hi=s.get("maxLength", INF))
            else:
                n = Node({"integer": "int", "number": "num", "boolean": "bool", "null": "null"}[t])
            out.append(n)
        if u is None:
            memo[id(s)] = out[0]
            return out[0]
        u.alts = out
        return u

    root = node(schema)
    # flatten unions, then the least document depth of every node (a fixpoint)
    allnodes, todo = [], [root]
    while todo:
        n = todo.pop()
        if any(n is m for m in allnodes):
            continue
        allnodes.append(n)
        if n.kind == "union":
            flat, stack = [], list(n.alts)
            while stack:
                a = stack.pop(0)
                if a.kind == "union":
                    stack = a.alts + stack
                elif not any(a is f for f in flat):
                    flat.append(a)
            n.alts = flat
            todo += flat
        elif n.kind == "obj":
            todo += [v for _, v in n.props]
        elif n.kind == "arr":
            todo.append(n.items)
    changed = True
    while changed:
        changed = False
        for n in allnodes:
            if n.kind == "objany":
                m = 1
            elif n.kind == "obj":
                m = 1 + max([v.mind for _, v in n.props[: n.nreq]], default=0)
            elif n.kind == "arr":
                m = 1 + (n.items.mind if n.lo > 0 else 0)
            elif n.kind == "union":
                m = min(a.mind for a in n.alts)
            else:
                m = 0
            m = min(m, INF)
            if m < n.mind:
                n.mind, changed = m, True
    return root


FIRST = {"any": b'{["-0123456789tfn', "objany": b"{", "obj": b"{", "arr": b"[", "str": b'"', "int": b"-0123456789",
         "num": b"-0123456789", "bool": b"tf", "null": b"n"}


def _first(n, c):
    if n.kind == "enum":
        return any(l[0] == c for l in n.lits)
    return c in FIRST[n.kind]


def _need(n, c):
    if n.kind == "any":
        return 1 if c in b"{[" else 0
    return n.mind


class _Ctx:
    closed = False


def _ws(c):
    if c == 0x20:
        return (yield)
    if c == 0x0A:
        k, c = 0, (yield)
        while c in (0x20, 0x09) and k < J.WS_MAX:
            k, c = k + 1, (yield)
    return c


def _string_body(hi=INF, on_byte=None):
    """after the opening quote, through the closing one; -> code points"""
    state, count = (J.STR, 0, 0, 0, 0, 0), 0
    while True:
        c = yield
        if on_byte:
            on_byte(c)
        if state[0] == J.STR and c == ord('"'):
            return count
        if state[0] == J.STR and (c < 0x80 or c >= 0xC0):
            if count >= hi:
                raise Reject
            count += 1
        state = J.step(state, c)
        if state is None:
            raise Reject


def _number(c, integer=False, on_byte=None):
    """c: the first byte; -> the byte after the number"""
    mode = {ord("-"): J.NUM_MINUS, ord("0"): J.NUM_ZERO}.get(c, J.NUM_INT)
    while True:
        c = yield
        if integer and c in b".eE":
            raise Reject
        nxt = J.NUM_NEXT[mode].get(c)
        if nxt is None:
            if mode in (J.NUM_MINUS, J.NUM_DOT, J.NUM_E, J.NUM_ESIGN):
                raise Reject
            return c
        if on_byte:
            on_byte(c)
        mode = nxt


def _literal(word, on_byte=None):
    for b in word[1:]:
        c = yield
        if on_byte:
            on_byte(c)
        if c != b:
            raise Reject


def _any(c, d, ctx):
    if c in b"{[":
        if d >= MAX_DEPTH:
            raise Reject
        close = ord("}") if c == ord("{") else ord("]")
        c = yield from _ws((yield))
        if c != close:
            while True:
                if close == ord("}"):
                    if c != ord('"'):
                        raise Reject
                    yield from _string_body()
                    c = yield from _ws((yield))
                    if c != ord(":"):
                        raise Reject
                    c = yield from _ws((yield))
                c = yield from _value(Node("any"), c, d + 1, ctx)
                if c == ord(","):
                    c = yield from _ws((yield))
                    continue
                if c != close:
                    raise Reject
                break
        if d == 0:
            ctx.closed = True
        return (yield from _ws((yield)))
    if c == ord('"'):
        yield from _string_body()
        return (yield from _ws((yield)))
    if c in b"-0123456789":
        return (yield from _ws((yield from _number(c))))
    for w in (b"true", b"false", b"null"):
        if c == w[0]:
            yield from _literal(w)
            return (yield from _ws((yield)))
    raise Reject


def _value(n, c, d, ctx):
    """c: the first byte of a value of n at depth d; consumes the value and its ws; -> the byte after"""
    if n.kind == "union":
        alts = [a for a in n.alts if _first(a, c)]
        if not alts:
            raise Reject
        n = alts[0]
    if not _first(n, c) or d + _need(n, c) > MAX_DEPTH:
        raise Reject
    if n.kind in ("any", "objany", "bool", "null"):
        return (yield from _any(c, d, ctx))
    if n.kind == "str":
        count = yield from _string_body(n.hi)
        if count < n.lo:
            raise Reject
        return (yield from _ws((yield)))
    if n.kind in ("int", "num"):
        return (yield from _ws((yield from _number(c, n.kind == "int"))))
    if n.kind == "enum":
        buf = bytearray([c])
        cands = [l for l in n.lits if l.startswith(bytes(buf))]

        def on_byte(b):
            buf.append(b)
            if not any(l.startswith(bytes(buf)) for l in cands):
                raise Reject
        if c == ord('"'):
            yield from _string_body(on_byte=on_byte)
            nxt = yield
        elif c in b"-0123456789":
            nxt = yield from _number(c, on_byte=on_byte)
        else:
            yield from _literal(next(l for l in cands), on_byte=on_byte)
            nxt = yield
        if bytes(buf) not in n.lits:
            raise Reject
        return (yield from _ws(nxt))
    if n.kind == "arr":
        di = d + 1
        fits = lambda k: k < n.hi and di + n.items.mind <= MAX_DEPTH
        c = yield from _ws((yield))
        count = 0
        if c == ord("]"):
            if n.lo > 0:
                raise Reject
        else:
            while True:
                if not fits(count):
                    raise Reject
                c = yield from _value(n.items, c, di, ctx)
                count += 1
                if c == ord(","):
                    if not fits(count):
                        raise Reject
                    c = yield from _ws((yield))
                    continue
                if c != ord("]") or count < n.lo:
                    raise Reject
                break
        return (yield from _ws((yield)))
    # an object with properties
    di = d + 1
    allowed = lambda p: [p] if p < n.nreq else [j for j in range(p, len(n.props)) if di + n.props[j][1].mind <= MAX_DEPTH]
    c = yield from _ws((yield))
    p = 0
    if c != ord("}"):
        while True:
            cands = allowed(p)
            if c != ord('"') or not cands:
                raise Reject
            buf = bytearray()

            def on_byte(b):
                buf.append(b)
                cands[:] = [j for j in cands if n.props[j][0].startswith(bytes(buf))]
                if not cands:
                    raise Reject
            yield from _string_body(on_byte=on_byte)
            k = next(j for j in cands if n.props[j][0] == bytes(buf))
            p = k + 1
            c = yield from _ws((yield))
            if c != ord(":"):
                raise Reject
            c = yield from _ws((yield))
            c = yield from _value(n.props[k][1], c, di, ctx)
            if c == ord(","):
                if not allowed(p):
                    raise Reject
                c = yield from _ws((yield))
                continue
            if c != ord("}"):
                raise Reject
            break
    if p < n.nreq:
        raise Reject
    if d == 0:
        ctx.closed = True
    return (yield from _ws((yield)))


def _doc(root, ctx):
    c = yield
    if c != ord("{"):
        raise Reject
    yield from _value(root, c, 0, ctx)
    raise Reject                                      # a byte that is not ws after the root


def run(root, data):
    """(viable, complete) of the bytes"""
    ctx = _Ctx()
    g = _doc(root, ctx)
    next(g)
    try:
        for c in bytes(data):
            g.send(c)
    except Reject:
        return False, False
    return True, ctx.closed


def viable(root, data):
    return run(root, data)[0]


def complete(root, data):
    return run(root, data)[1]


def mask(root, pieces, stop_ids, generated):
    """bool[n_vocab]: the tokens the draw after `generated` may take"""
    import numpy as np
    stops = set(int(s) for s in stop_ids)
    prefix = b"".join(pieces[int(t)] for t in generated)
    ok, done = run(root, prefix)
    assert ok, "the history is not a viable prefix"
    out = np.zeros(len(pieces), dtype=bool)
    for t, pc in enumerate(pieces):
        out[t] = done if t in stops else (bool(pc) and viable(root, prefix + pc))
    return out


def apply_mask(root, logits, pieces, stop_ids, generated):
    import numpy as np
    out = np.array(logits, dtype=np.float32, copy=True)
    out[~mask(root, pieces, stop_ids, generated)] = -np.inf
    return out
