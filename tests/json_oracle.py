"""TEST INFRASTRUCTURE: the JSON language of `format: "json"` (include/gridllm_native.h, gl_sample_opts.format) restated in
Python, and the mask it implies over a vocabulary.

    root    ::= object
    value   ::= object | array | string | number | ("true" | "false" | "null") ws
    object  ::= "{" ws ( string ":" ws value ( "," ws string ":" ws value )* )? "}" ws
    array   ::= "[" ws ( value ( "," ws value )* )? "]" ws
    string  ::= "\\"" ( char | "\\\\" ( ["\\\\/bfnrt] | "u" hex hex hex hex ) )* "\\"" ws
    char    ::= any Unicode scalar value >= U+0020 other than " and \\, as well-formed UTF-8
    number  ::= "-"? ( "0" | [1-9] [0-9]* ) ( "." [0-9]+ )? ( [eE] [-+]? [0-9]+ )? ws
    ws      ::= "" | " " | "\\n" [ \\t]{0,20}

Nesting depth <= 64, root included.  A stop token is allowed exactly when the root object has closed (anywhere in its trailing
ws); control tokens (empty piece) never; any other token when every byte of its piece is accepted.

The state is a tuple (mode, depth, stack, cnt, aux, key) with the meaning json_fsm.h gives its JsonState fields, so that the
device automaton can be compared with this one state for state (tests/test_json_cpu.py); the code is written independently."""
import numpy as np

MAX_DEPTH = 64
WS_MAX = 20
WS_CLOSED = WS_MAX + 2

(START, OBJ_FIRST, OBJ_KEY, COLON, VALUE, ARR_FIRST, AFTER, STR, STR_ESC, STR_HEX, STR_UTF8, NUM_MINUS, NUM_ZERO, NUM_INT, NUM_DOT,
 NUM_FRAC, NUM_E, NUM_ESIGN, NUM_EXP, LIT) = range(20)
WS_MODES = (OBJ_FIRST, OBJ_KEY, COLON, VALUE, ARR_FIRST, AFTER)
LITERALS = (b"true", b"false", b"null")
# ranges of the next UTF-8 continuation byte (RFC 3629 table 3-7): aux codes of json_fsm.h
CONT_RANGES = {0: (0x80, 0xBF), 1: (0xA0, 0xBF), 2: (0x80, 0x9F), 3: (0x90, 0xBF), 4: (0x80, 0x8F)}
# lead byte -> (continuation bytes, aux of the first one)
LEADS = {**{b: (1, 0) for b in range(0xC2, 0xE0)}, 0xE0: (2, 1), **{b: (2, 0) for b in range(0xE1, 0xED)}, 0xED: (2, 2),
         0xEE: (2, 0), 0xEF: (2, 0), 0xF0: (3, 3), 0xF1: (3, 0), 0xF2: (3, 0), 0xF3: (3, 0), 0xF4: (3, 4)}
INITIAL = (START, 0, 0, 0, 0, 0)
DIGITS = frozenset(b"0123456789")
HEX = frozenset(b"0123456789abcdefABCDEF")
# what may follow each part of a number
NUM_NEXT = {
    NUM_MINUS: {**{d: NUM_INT for d in b"123456789"}, ord("0"): NUM_ZERO},
    NUM_ZERO: {ord("."): NUM_DOT, ord("e"): NUM_E, ord("E"): NUM_E},
    NUM_INT: {**{d: NUM_INT for d in DIGITS}, ord("."): NUM_DOT, ord("e"): NUM_E, ord("E"): NUM_E},
    NUM_DOT: {d: NUM_FRAC for d in DIGITS},
    NUM_FRAC: {**{d: NUM_FRAC for d in DIGITS}, ord("e"): NUM_E, ord("E"): NUM_E},
    NUM_E: {**{d: NUM_EXP for d in DIGITS}, ord("+"): NUM_ESIGN, ord("-"): NUM_ESIGN},
    NUM_ESIGN: {d: NUM_EXP for d in DIGITS},
    NUM_EXP: {d: NUM_EXP for d in DIGITS},
}


def _top_is_object(depth, stack):
    return bool((stack >> (depth - 1)) & 1)


def _open(depth, stack, aux, obj):
    if depth >= MAX_DEPTH:
        return None
    stack = stack | (1 << depth) if obj else stack & ~(1 << depth)
    return (OBJ_FIRST if obj else ARR_FIRST, depth + 1, stack, 0, aux, 0)


def _value(depth, stack, aux, c):
    """first byte of a value; None when no value starts with it"""
    if c == ord("{"):
        return _open(depth, stack, aux, True)
    if c == ord("["):
        return _open(depth, stack, aux, False)
    if c == ord('"'):
        return (STR, depth, stack, 0, aux, 0)
    if c == ord("-"):
        return (NUM_MINUS, depth, stack, 0, aux, 0)
    if c == ord("0"):
        return (NUM_ZERO, depth, stack, 0, aux, 0)
    if c in DIGITS:
        return (NUM_INT, depth, stack, 0, aux, 0)
    for i, lit in enumerate(LITERALS):
        if c == lit[0]:
            return (LIT, depth, stack, 1, i, 0)
    return None


def step(state, c):
    """state after byte c, or None when c takes the text outside the language"""
    mode, depth, stack, cnt, aux, key = state
    if mode == START:
        return _open(0, stack, aux, True) if c == ord("{") else None
    if mode == STR:
        if c == ord('"'):
            return (COLON if key else AFTER, depth, stack, 0, aux, 0)
        if c == ord("\\"):
            return (STR_ESC, depth, stack, cnt, aux, key)
        if c < 0x20:
            return None
        if c < 0x80:
            return state
        if c in LEADS:
            n, a = LEADS[c]
            return (STR_UTF8, depth, stack, n, a, key)
        return None
    if mode == STR_UTF8:
        lo, hi = CONT_RANGES[aux]
        if not lo <= c <= hi:
            return None
        return (STR_UTF8 if cnt > 1 else STR, depth, stack, cnt - 1, 0, key)
    if mode == STR_ESC:
        if c in b'"\\/bfnrt':
            return (STR, depth, stack, cnt, aux, key)
        if c == ord("u"):
            return (STR_HEX, depth, stack, 4, aux, key)
        return None
    if mode == STR_HEX:
        if c not in HEX:
            return None
        return (STR_HEX if cnt > 1 else STR, depth, stack, cnt - 1, aux, key)
    if mode == LIT:
        lit = LITERALS[aux]
        if c != lit[cnt]:
            return None
        if cnt + 1 == len(lit):
            return (AFTER, depth, stack, 0, aux, key)
        return (LIT, depth, stack, cnt + 1, aux, key)
    # numbers: a byte that cannot continue one ends it and goes to the ws slot behind it
    if mode in NUM_NEXT:
        nxt = NUM_NEXT[mode].get(c)
        if nxt is not None:
            return (nxt, depth, stack, cnt, aux, key)
        if mode in (NUM_MINUS, NUM_DOT, NUM_E, NUM_ESIGN):     # the number is not complete yet
            return None
        mode, cnt = AFTER, 0
    # a ws slot: "" | " " | "\n" [ \t]{0,20}
    if c == ord(" "):
        if cnt == 0:
            return (mode, depth, stack, WS_CLOSED, aux, key)
        return (mode, depth, stack, cnt + 1, aux, key) if 1 <= cnt <= WS_MAX else None
    if c == ord("\t"):
        return (mode, depth, stack, cnt + 1, aux, key) if 1 <= cnt <= WS_MAX else None
    if c == ord("\n"):
        return (mode, depth, stack, 1, aux, key) if cnt == 0 else None
    if mode == OBJ_FIRST and c == ord("}"):
        return (AFTER, depth - 1, stack, 0, aux, key)
    if mode in (OBJ_FIRST, OBJ_KEY):
        return (STR, depth, stack, 0, aux, 1) if c == ord('"') else None
    if mode == COLON:
        return (VALUE, depth, stack, 0, aux, key) if c == ord(":") else None
    if mode == ARR_FIRST and c == ord("]"):
        return (AFTER, depth - 1, stack, 0, aux, key)
    if mode in (VALUE, ARR_FIRST):
        return _value(depth, stack, aux, c)
    if mode == AFTER and depth > 0:
        obj = _top_is_object(depth, stack)
        if c == ord(","):
            return (OBJ_KEY if obj else VALUE, depth, stack, 0, aux, key)
        if c == ord("}" if obj else "]"):
            return (AFTER, depth - 1, stack, 0, aux, key)
    return None


def run(data, state=INITIAL):
    """state after the bytes, or None"""
    for c in bytes(data):
        state = step(state, c)
        if state is None:
            return None
    return state


def done(state):
    return state is not None and state[0] == AFTER and state[1] == 0


def viable(data):
    """the bytes are a prefix of some document of the language"""
    return run(data) is not None


def complete(data):
    """the bytes are a whole document: a stop token may follow"""
    return done(run(data))


def token_allowed(state, piece, is_stop):
    if is_stop:
        return done(state)
    if not piece:
        return False
    return run(piece, state) is not None


def mask(pieces, stop_ids, generated):
    """bool[n_vocab]: the tokens the draw after `generated` may take (pieces[t]: bytes of token t)"""
    stops = set(int(s) for s in stop_ids)
    state = run(b"".join(pieces[int(t)] for t in generated))
    assert state is not None, "the history is not a viable prefix"
    return np.array([token_allowed(state, pieces[t], t in stops) for t in range(len(pieces))], dtype=bool)


def apply_mask(logits, pieces, stop_ids, generated):
    out = np.array(logits, dtype=np.float32, copy=True)
    out[~mask(pieces, stop_ids, generated)] = -np.inf
    return out
