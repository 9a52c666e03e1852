// Byte-level automaton of the language a registered JSON schema defines (include/gridllm_native.h, gl_format_schema; compiled
// by schema_compile.cpp; restated in tests/schema_oracle.py).  It layers over the JSON automaton of json_fsm.h: every byte runs
// through json_step, which keeps JsonState with its fields and meaning (syntax, ws, nesting), and the schema layer refuses the
// bytes a schema rules out.  The layer holds
//   - a cursor: the node of the value being read, the literal candidate and the bytes (or code points) matched so far;
//   - one frame per open container of the schema: its node and its progress (objects: the next property index; arrays: the
//     items completed).
// A container of an unconstrained value (node kind SK_ANY / SK_OBJ_ANY) pushes no frame: the cursor's phase SP_ANY hands the
// whole value to json_step and remembers the depth it started at.
//
// Keys and enum members are matched byte by byte against literals in canonical spelling (keys carry their closing quote).
// The candidates of a match are ordered and distinct, so the cursor keeps the lowest candidate still consistent with the bytes
// read and the count matched; the next byte moves it to the lowest candidate with the same prefix and that byte next.
//
// No dead ends: every node carries the least nesting depth of a document of it (mind), and the automaton only opens a
// container, picks an optional key or starts an array item when a document of it still closes within JSON_MAX_DEPTH.
//
// The frames are reached through an accessor F (F::at(d) = the frame at index d, an lvalue; it is only ever asked for the frame
// on top of the stack or one just pushed), so the mask kernel can walk a piece over a private overlay of the frames it touches
// while the others stay in shared memory (schema_mask.cu), and the host runs the same code over a plain array.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "json_fsm.h"

namespace gl {

constexpr int SCHEMA_MAX_NODES = 4096;
constexpr int SCHEMA_MAX_PROPS = 255;
constexpr uint16_t SCHEMA_UNBOUNDED = 0xFFFF;     // a maximum that is absent; counters saturate here
constexpr uint8_t SCHEMA_INF = 255;               // mind of a node without a finite document

enum : uint8_t {
    SK_ANY = 0,      // any value of the JSON language
    SK_OBJ_ANY,      // any object
    SK_OBJ,          // object with properties: n props at list[2i] (key literal), list[2i + 1] (value node); lo required ones first
    SK_ARR,          // array: items node = list (SK_ANY when absent); lo / hi: minItems / maxItems
    SK_STR,          // string: lo / hi: minLength / maxLength in code points (an escape counts as one)
    SK_INT,          // -? (0 | [1-9][0-9]*)
    SK_NUM,          // the number of the JSON language
    SK_BOOL,
    SK_NULL,
    SK_ENUM,         // n literals (ids at list[i]), ordered and distinct
    SK_UNION,        // n alternatives (node ids at list[i]), none a union, with disjoint sets of first bytes
};

struct SchemaNode {      // 16 bytes
    uint8_t kind, mind;
    uint16_t n;
    uint16_t lo, hi;
    uint32_t list;
    uint32_t pad;
};
static_assert(sizeof(SchemaNode) == 16, "SchemaNode is 16 bytes");

// a compiled schema is one blob: this header, then the tables at the byte offsets it gives
struct SchemaHeader {
    uint32_t root, n_nodes, n_list, n_lits;
    uint32_t off_nodes, off_list, off_lit_off, off_lit;
};

struct SchemaView {
    const SchemaNode* nodes;
    const uint16_t* list;
    const uint32_t* lit_off;     // [n_lits + 1]
    const uint8_t* lit;
    uint32_t root;
};

JSON_HD SchemaView schema_view(const uint8_t* blob) {
    const SchemaHeader* h = reinterpret_cast<const SchemaHeader*>(blob);
    SchemaView v;
    v.nodes = reinterpret_cast<const SchemaNode*>(blob + h->off_nodes);
    v.list = reinterpret_cast<const uint16_t*>(blob + h->off_list);
    v.lit_off = reinterpret_cast<const uint32_t*>(blob + h->off_lit_off);
    v.lit = blob + h->off_lit;
    v.root = h->root;
    return v;
}

enum : uint8_t {
    SP_VALUE = 0,    // a value of cur.node is next (json modes START / VALUE)
    SP_CONT,         // between the parts of the schema container on top (or after the root)
    SP_KEY,          // a key of the object on top: candidate cand, n bytes matched
    SP_STR,          // a string of cur.node: n code points so far
    SP_NUM,          // a number of cur.node
    SP_ENUM,         // a member of the enum cur.node: candidate cand, n bytes matched
    SP_ANY,          // an unconstrained value that started at depth base
};

struct SchemaCursor {    // 8 bytes
    uint16_t node, cand, n;
    uint8_t phase, base;
};
struct SchemaFrame {     // 4 bytes
    uint16_t node, prog;
};

// 16 + 8 + 4 * 64 bytes
struct SchemaState {
    JsonState js;
    SchemaCursor cur;
    SchemaFrame fr[JSON_MAX_DEPTH];
};
static_assert(sizeof(SchemaState) == 280, "SchemaState is 280 bytes");

struct SchemaArrayFrames {       // the host's accessor: the frames of a whole state
    SchemaFrame* a;
    JSON_HD SchemaFrame& at(int d) { return a[d]; }
};

JSON_HD void schema_init(JsonState& js, SchemaCursor& cur, const SchemaView& v) {
    js = JsonState{};
    cur = SchemaCursor{};
    cur.node = (uint16_t)v.root;
    cur.phase = SP_VALUE;
}

JSON_HD uint32_t schema_lit_len(const SchemaView& v, int lit) { return v.lit_off[lit + 1] - v.lit_off[lit]; }
JSON_HD uint8_t schema_lit_byte(const SchemaView& v, int lit, int i) { return v.lit[v.lit_off[lit] + i]; }

// the byte a value of node k (not a union) can start with
JSON_HD bool schema_first_ok(const SchemaView& v, int k, uint8_t c) {
    const SchemaNode& nd = v.nodes[k];
    switch (nd.kind) {
        case SK_ANY:
            return c == '{' || c == '[' || c == '"' || c == '-' || json_is_digit(c) || c == 't' || c == 'f' || c == 'n';
        case SK_OBJ_ANY:
        case SK_OBJ: return c == '{';
        case SK_ARR: return c == '[';
        case SK_STR: return c == '"';
        case SK_INT:
        case SK_NUM: return c == '-' || json_is_digit(c);
        case SK_BOOL: return c == 't' || c == 'f';
        case SK_NULL: return c == 'n';
        case SK_ENUM:
            for (int i = 0; i < nd.n; ++i)
                if (schema_lit_byte(v, v.list[nd.list + i], 0) == c) return true;
            return false;
        default: return false;
    }
}

// least nesting depth a value of node k that starts with byte c needs
JSON_HD int schema_need(const SchemaView& v, int k, uint8_t c) {
    const SchemaNode& nd = v.nodes[k];
    if (nd.kind == SK_ANY) return (c == '{' || c == '[') ? 1 : 0;
    return nd.mind;
}

// Literal match: the lowest candidate j in [cand, hi) whose first n bytes equal those of cand and whose byte n is c (c < 0:
// whose length is n).  ids(j) = the literal of candidate j; ok(j) = the candidate may be taken at all.  -1: none.
template <class Ids, class Ok>
JSON_HD int schema_match(const SchemaView& v, int cand, int hi, int n, int c, Ids ids, Ok ok) {
    const int lc = ids(cand);
    for (int j = cand; j < hi; ++j) {
        if (!ok(j)) continue;
        const int lj = ids(j);
        const int len = (int)schema_lit_len(v, lj);
        if (c < 0 ? len != n : (len <= n || schema_lit_byte(v, lj, n) != (uint8_t)c)) continue;
        bool same = true;
        for (int i = 0; i < n && same; ++i) same = schema_lit_byte(v, lj, i) == schema_lit_byte(v, lc, i);
        if (same) return j;
    }
    return -1;
}

// the object on top (node o, at depth d) may take property j as its next key
JSON_HD bool schema_key_fits(const SchemaView& v, const SchemaNode& o, int j, int d) {
    return d + v.nodes[v.list[o.list + 2 * j + 1]].mind <= JSON_MAX_DEPTH;
}

// the lowest key the object on top may take next (progress p), or -1
JSON_HD int schema_first_key(const SchemaView& v, const SchemaNode& o, int p, int d) {
    if (p < o.lo) return p;                                      // a required key: it fits, or the object would not have opened
    for (int j = p; j < o.n; ++j)
        if (schema_key_fits(v, o, j, d)) return j;
    return -1;
}

// one more item may start in the array on top (node a, at depth d, prog items done)
JSON_HD bool schema_item_fits(const SchemaView& v, const SchemaNode& a, int prog, int d) {
    return prog < a.hi && d + v.nodes[a.list].mind <= JSON_MAX_DEPTH;
}

// a value at the schema level ended: the array around it counts it
template <class F>
JSON_HD void schema_value_done(JsonState& js, SchemaCursor& cur, F& fr) {
    cur.phase = SP_CONT;
    if (js.depth > 0 && !json_top_is_object(js)) {
        SchemaFrame& f = fr.at(js.depth - 1);
        if (f.prog < SCHEMA_UNBOUNDED) ++f.prog;
    }
}

// the first byte of a value of node k (json modes START / VALUE / ARR_FIRST, ws already handled)
template <class F>
JSON_HD bool schema_begin_value(const SchemaView& v, JsonState& js, SchemaCursor& cur, F& fr, int k, uint8_t c) {
    if (v.nodes[k].kind == SK_UNION) {
        const SchemaNode& u = v.nodes[k];
        int pick = -1;
        for (int i = 0; i < u.n && pick < 0; ++i)
            if (schema_first_ok(v, v.list[u.list + i], c)) pick = v.list[u.list + i];
        if (pick < 0) return false;
        k = pick;
    }
    if (!schema_first_ok(v, k, c)) return false;
    const int d0 = js.depth;
    if (d0 + schema_need(v, k, c) > JSON_MAX_DEPTH) return false;
    if (!json_step(js, c)) return false;
    const SchemaNode& nd = v.nodes[k];
    cur.node = (uint16_t)k;
    cur.n = 0;
    switch (nd.kind) {
        case SK_OBJ:
        case SK_ARR: {
            SchemaFrame& f = fr.at(d0);
            f.node = (uint16_t)k;
            f.prog = 0;
            cur.phase = SP_CONT;
            return true;
        }
        case SK_STR: cur.phase = SP_STR; return true;
        case SK_INT:
        case SK_NUM: cur.phase = SP_NUM; return true;
        case SK_ENUM: {
            const int j = schema_match(v, 0, nd.n, 0, c, [&](int i) { return (int)v.list[nd.list + i]; }, [](int) { return true; });
            cur.cand = (uint16_t)j;
            cur.n = 1;
            cur.phase = SP_ENUM;
            return true;
        }
        default: cur.phase = SP_ANY; cur.base = (uint8_t)d0; return true;      // any value / object, booleans, null
    }
}

// One byte.  false: the byte takes the generated text outside the schema's language (the state is then unspecified).
template <class F>
JSON_HD bool schema_step(const SchemaView& v, JsonState& js, SchemaCursor& cur, F& fr, uint8_t c) {
    // a number ends on a byte that cannot continue it; the byte then belongs to the ws slot behind it (as in json_step)
    const uint8_t m = js.mode;
    if (m == JM_NUM_ZERO || m == JM_NUM_INT || m == JM_NUM_FRAC || m == JM_NUM_EXP) {
        const bool more = (json_is_digit(c) && m != JM_NUM_ZERO) || (c == '.' && (m == JM_NUM_ZERO || m == JM_NUM_INT)) ||
                          ((c == 'e' || c == 'E') && m != JM_NUM_EXP);
        if (!more) {
            if (cur.phase == SP_ENUM) {
                const SchemaNode& nd = v.nodes[cur.node];
                const int j = schema_match(v, cur.cand, nd.n, cur.n, -1, [&](int i) { return (int)v.list[nd.list + i]; }, [](int) { return true; });
                if (j < 0) return false;
                cur.cand = (uint16_t)j;
                js.mode = JM_AFTER; js.cnt = 0;
                schema_value_done(js, cur, fr);
            } else if (cur.phase == SP_NUM || (cur.phase == SP_ANY && js.depth == cur.base)) {
                js.mode = JM_AFTER; js.cnt = 0;
                schema_value_done(js, cur, fr);
            }
        } else if (cur.phase == SP_NUM && v.nodes[cur.node].kind == SK_INT && !json_is_digit(c)) {
            return false;                                            // an integer has no fraction and no exponent
        }
    }
    switch (cur.phase) {
        case SP_ANY:
            if (!json_step(js, c)) return false;
            if (js.depth == cur.base && js.mode == JM_AFTER) schema_value_done(js, cur, fr);
            return true;
        case SP_NUM:
            return json_step(js, c);
        case SP_STR: {
            const SchemaNode& nd = v.nodes[cur.node];
            if (js.mode == JM_STR) {
                if (c == '"') {
                    if (cur.n < nd.lo || !json_step(js, c)) return false;
                    schema_value_done(js, cur, fr);
                    return true;
                }
                if (c < 0x80 || c >= 0xC0) {                         // a new character (or escape) starts
                    if (nd.hi != SCHEMA_UNBOUNDED && cur.n >= nd.hi) return false;
                    if (cur.n < SCHEMA_UNBOUNDED) ++cur.n;
                }
            }
            return json_step(js, c);
        }
        case SP_ENUM: {
            const SchemaNode& nd = v.nodes[cur.node];
            const int j = schema_match(v, cur.cand, nd.n, cur.n, c, [&](int i) { return (int)v.list[nd.list + i]; }, [](int) { return true; });
            if (j < 0) return false;
            const int d0 = js.depth;
            if (!json_step(js, c)) return false;
            cur.cand = (uint16_t)j;
            ++cur.n;
            if (js.mode == JM_AFTER && js.depth == d0) {            // a string or true / false / null closed
                if (cur.n != schema_lit_len(v, v.list[nd.list + j])) return false;
                schema_value_done(js, cur, fr);
            }
            return true;
        }
        case SP_KEY: {
            SchemaFrame& f = fr.at(js.depth - 1);
            const SchemaNode& o = v.nodes[f.node];
            const int hi = f.prog < o.lo ? f.prog + 1 : o.n;
            const int d = js.depth;
            const int j = schema_match(v, cur.cand, hi, cur.n, c, [&](int i) { return (int)v.list[o.list + 2 * i]; },
                                       [&](int i) { return i < o.lo || schema_key_fits(v, o, i, d); });
            if (j < 0) return false;
            const bool closing = js.mode == JM_STR && c == '"';
            if (!json_step(js, c)) return false;
            cur.cand = (uint16_t)j;
            ++cur.n;
            if (closing) {                                           // the key is j: its value comes next
                f.prog = (uint16_t)(j + 1);
                cur.node = v.list[o.list + 2 * j + 1];
                cur.phase = SP_CONT;
            }
            return true;
        }
        case SP_VALUE:
            if (js.mode != JM_START && (c == ' ' || c == '\t' || c == '\n')) return json_step(js, c);
            if (js.mode == JM_START && c != '{') return false;
            return schema_begin_value(v, js, cur, fr, cur.node, c);
        default:
            break;
    }
    // SP_CONT: between the parts of the container on top
    if (c == ' ' || c == '\t' || c == '\n' || js.depth == 0) return json_step(js, c);
    SchemaFrame& f = fr.at(js.depth - 1);
    const SchemaNode& nd = v.nodes[f.node];
    const int d = js.depth;
    switch (js.mode) {
        case JM_OBJ_FIRST:
        case JM_OBJ_KEY:
            if (c == '}') {
                if (js.mode != JM_OBJ_FIRST || f.prog < nd.lo || !json_step(js, c)) return false;
                schema_value_done(js, cur, fr);
                return true;
            }
            if (c == '"') {
                const int j = schema_first_key(v, nd, f.prog, d);
                if (j < 0 || !json_step(js, c)) return false;
                cur.phase = SP_KEY;
                cur.cand = (uint16_t)j;
                cur.n = 0;
                return true;
            }
            return false;
        case JM_COLON:
            if (!json_step(js, c)) return false;
            cur.phase = SP_VALUE;
            return true;
        case JM_ARR_FIRST:
            if (c == ']') {
                if (nd.lo > 0 || !json_step(js, c)) return false;
                schema_value_done(js, cur, fr);
                return true;
            }
            if (!schema_item_fits(v, nd, 0, d)) return false;
            return schema_begin_value(v, js, cur, fr, nd.list, c);
        case JM_AFTER: {
            const bool obj = json_top_is_object(js);
            if (c == ',') {
                if (obj ? schema_first_key(v, nd, f.prog, d) < 0 : !schema_item_fits(v, nd, f.prog, d)) return false;
                if (!json_step(js, c)) return false;
                if (!obj) { cur.phase = SP_VALUE; cur.node = (uint16_t)nd.list; }
                return true;
            }
            if (c == (obj ? '}' : ']')) {
                if (f.prog < nd.lo || !json_step(js, c)) return false;
                schema_value_done(js, cur, fr);
                return true;
            }
            return false;
        }
        default:
            return false;
    }
}

JSON_HD bool schema_done(const JsonState& js) { return json_done(js); }

template <class F>
JSON_HD bool schema_run(const SchemaView& v, JsonState& js, SchemaCursor& cur, F& fr, const uint8_t* p, int n) {
    for (int i = 0; i < n; ++i)
        if (!schema_step(v, js, cur, fr, p[i])) return false;
    return true;
}

// host: schema_utf8[0..n) -> blob; GL_OK, or GL_ERR_INVALID (malformed JSON) / GL_ERR_UNSUPPORTED (outside the subset) with a
// message naming the keyword and its JSON pointer (schema_compile.cpp)
int schema_compile(const char* schema_utf8, size_t n, std::vector<uint8_t>& blob, std::string& err);

}  // namespace gl
