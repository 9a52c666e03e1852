// Byte-level automaton of the JSON language a request with `format: "json"` is held to (include/gridllm_native.h,
// gl_sample_opts.format; restated in tests/json_oracle.py):
//
//   root    ::= object
//   value   ::= object | array | string | number | ("true" | "false" | "null") ws
//   object  ::= "{" ws ( string ":" ws value ( "," ws string ":" ws value )* )? "}" ws
//   array   ::= "[" ws ( value ( "," ws value )* )? "]" ws
//   string  ::= "\"" ( char | "\\" ( ["\\/bfnrt] | "u" hex hex hex hex ) )* "\"" ws
//   char    ::= a Unicode scalar value >= U+0020 other than " and \, as well-formed UTF-8
//   number  ::= "-"? ( "0" | [1-9] [0-9]* ) ( "." [0-9]+ )? ( [eE] [-+]? [0-9]+ )? ws
//   ws      ::= "" | " " | "\n" [ \t]{0,20}
//
// with nesting depth <= JSON_MAX_DEPTH (root included).  The grammar never puts two ws slots side by side, so one counter
// tracks the current slot.  Everything is __host__ __device__: the mask kernel (schema_mask.cu) runs exactly this program per
// vocabulary entry, the host validates histories with it (gl_constrain_logits), and tests/test_json_cpu.py compiles it with g++
// and checks it state for state against the Python restatement.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define JSON_HD __host__ __device__ __forceinline__
#else
#define JSON_HD inline
#endif

namespace gl {

constexpr int JSON_MAX_DEPTH = 64;
constexpr int JSON_WS_MAX = 20;          // [ \t] after a newline

// modes; the first six are the ones with a ws slot in front of what they expect (cnt = the slot's whitespace so far)
enum : uint8_t {
    JM_START = 0,      // nothing generated: '{'
    JM_OBJ_FIRST,      // after '{': '"' or '}'
    JM_OBJ_KEY,        // after ',' in an object: '"'
    JM_COLON,          // after a key: ':'
    JM_VALUE,          // after ':' or after ',' in an array: a value
    JM_ARR_FIRST,      // after '[': a value or ']'
    JM_AFTER,          // after a value: ',' or the container's closer; at depth 0 (the root closed): nothing but ws
    JM_STR,            // string body
    JM_STR_ESC,        // after '\'
    JM_STR_HEX,        // \u: cnt hex digits to go
    JM_STR_UTF8,       // cnt continuation bytes to go, the next one in range aux
    JM_NUM_MINUS,      // '-': a digit
    JM_NUM_ZERO,       // a leading 0: '.', e / E or the end
    JM_NUM_INT,        // [1-9][0-9]*: a digit, '.', e / E or the end
    JM_NUM_DOT,        // '.': a digit
    JM_NUM_FRAC,       // fraction digits: a digit, e / E or the end
    JM_NUM_E,          // e / E: a sign or a digit
    JM_NUM_ESIGN,      // exponent sign: a digit
    JM_NUM_EXP,        // exponent digits: a digit or the end
    JM_LIT,            // true / false / null: literal aux, cnt bytes matched
    JM_N_MODES
};

// ws slot counter: 0 nothing yet, 1 + k: "\n" and k of [ \t] (k <= 20), JSON_WS_CLOSED: " " (nothing more fits)
constexpr uint8_t JSON_WS_CLOSED = 2 + JSON_WS_MAX;
// the allowed range of the next UTF-8 continuation byte (RFC 3629: no overlong forms, no surrogates, nothing above U+10FFFF)
enum : uint8_t { JU_80_BF = 0, JU_A0_BF, JU_80_9F, JU_90_BF, JU_80_8F };

// 16 bytes; all zero is the initial state
struct JsonState {
    uint32_t stk_lo, stk_hi;     // bit d: the container at depth d + 1 is an object (1) or an array (0)
    uint8_t mode, depth, cnt, aux;
    uint8_t key;                 // the string being read is an object key
    uint8_t pad[3];
};
static_assert(sizeof(JsonState) == 16, "JsonState is 16 bytes");

JSON_HD bool json_top_is_object(const JsonState& s) {
    const int b = s.depth - 1;
    return ((b < 32 ? (s.stk_lo >> b) : (s.stk_hi >> (b - 32))) & 1u) != 0;
}

JSON_HD bool json_push(JsonState& s, bool object) {
    if (s.depth >= JSON_MAX_DEPTH) return false;
    const int b = s.depth;
    if (b < 32) s.stk_lo = object ? (s.stk_lo | (1u << b)) : (s.stk_lo & ~(1u << b));
    else s.stk_hi = object ? (s.stk_hi | (1u << (b - 32))) : (s.stk_hi & ~(1u << (b - 32)));
    s.depth = (uint8_t)(b + 1);
    s.mode = object ? JM_OBJ_FIRST : JM_ARR_FIRST;
    s.cnt = 0;
    return true;
}

JSON_HD void json_close(JsonState& s) {
    s.depth = (uint8_t)(s.depth - 1);
    s.mode = JM_AFTER;
    s.cnt = 0;
}

JSON_HD bool json_is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

// byte i of literal 0 "true", 1 "false", 2 "null" (packed little-endian; "false" keeps its 'f' outside the word)
JSON_HD uint8_t json_lit_char(int lit, int i) {
    if (lit == 1) return i == 0 ? (uint8_t)'f' : (uint8_t)(0x65736c61u >> (8 * (i - 1)));
    return (uint8_t)((lit == 0 ? 0x65757274u : 0x6c6c756eu) >> (8 * i));
}
JSON_HD int json_lit_len(int lit) { return lit == 1 ? 5 : 4; }

// the first byte of a value (modes VALUE / ARR_FIRST)
JSON_HD bool json_begin_value(JsonState& s, uint8_t c) {
    s.cnt = 0;
    switch (c) {
        case '{': return json_push(s, true);
        case '[': return json_push(s, false);
        case '"': s.mode = JM_STR; s.key = 0; return true;
        case '-': s.mode = JM_NUM_MINUS; return true;
        case '0': s.mode = JM_NUM_ZERO; return true;
        case 't': s.mode = JM_LIT; s.aux = 0; s.cnt = 1; return true;
        case 'f': s.mode = JM_LIT; s.aux = 1; s.cnt = 1; return true;
        case 'n': s.mode = JM_LIT; s.aux = 2; s.cnt = 1; return true;
        default:
            if (c >= '1' && c <= '9') { s.mode = JM_NUM_INT; return true; }
            return false;
    }
}

// One byte.  false: the byte takes the generated text outside the language (s is then unspecified).
JSON_HD bool json_step(JsonState& s, uint8_t c) {
    // ---- modes without a ws slot; a number that ends falls through to the ws slot behind it ----
    switch (s.mode) {
        case JM_START:
            return c == '{' && json_push(s, true);
        case JM_STR:
            if (c == '"') { s.mode = s.key ? JM_COLON : JM_AFTER; s.key = 0; s.cnt = 0; return true; }
            if (c == '\\') { s.mode = JM_STR_ESC; return true; }
            if (c < 0x20) return false;
            if (c < 0x80) return true;
            if (c >= 0xC2 && c <= 0xDF) { s.mode = JM_STR_UTF8; s.cnt = 1; s.aux = JU_80_BF; return true; }
            if (c >= 0xE0 && c <= 0xEF) {
                s.mode = JM_STR_UTF8; s.cnt = 2;
                s.aux = c == 0xE0 ? JU_A0_BF : c == 0xED ? JU_80_9F : JU_80_BF;
                return true;
            }
            if (c >= 0xF0 && c <= 0xF4) {
                s.mode = JM_STR_UTF8; s.cnt = 3;
                s.aux = c == 0xF0 ? JU_90_BF : c == 0xF4 ? JU_80_8F : JU_80_BF;
                return true;
            }
            return false;
        case JM_STR_UTF8: {
            const uint8_t lo = s.aux == JU_A0_BF ? 0xA0 : s.aux == JU_90_BF ? 0x90 : 0x80;
            const uint8_t hi = s.aux == JU_80_9F ? 0x9F : s.aux == JU_80_8F ? 0x8F : 0xBF;
            if (c < lo || c > hi) return false;
            s.aux = JU_80_BF;
            if (--s.cnt == 0) s.mode = JM_STR;
            return true;
        }
        case JM_STR_ESC:
            if (c == '"' || c == '\\' || c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't') { s.mode = JM_STR; return true; }
            if (c == 'u') { s.mode = JM_STR_HEX; s.cnt = 4; return true; }
            return false;
        case JM_STR_HEX:
            if (!(json_is_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'))) return false;
            if (--s.cnt == 0) s.mode = JM_STR;
            return true;
        case JM_LIT:
            if (c != json_lit_char(s.aux, s.cnt)) return false;
            if (++s.cnt == json_lit_len(s.aux)) { s.mode = JM_AFTER; s.cnt = 0; }
            return true;
        case JM_NUM_MINUS:
            if (c == '0') { s.mode = JM_NUM_ZERO; return true; }
            if (c >= '1' && c <= '9') { s.mode = JM_NUM_INT; return true; }
            return false;
        case JM_NUM_DOT:
            if (json_is_digit(c)) { s.mode = JM_NUM_FRAC; return true; }
            return false;
        case JM_NUM_E:
            if (c == '+' || c == '-') { s.mode = JM_NUM_ESIGN; return true; }
            if (json_is_digit(c)) { s.mode = JM_NUM_EXP; return true; }
            return false;
        case JM_NUM_ESIGN:
            if (json_is_digit(c)) { s.mode = JM_NUM_EXP; return true; }
            return false;
        case JM_NUM_ZERO:
        case JM_NUM_INT:
        case JM_NUM_FRAC:
        case JM_NUM_EXP:
            if (json_is_digit(c) && s.mode != JM_NUM_ZERO) return true;
            if (c == '.' && s.mode != JM_NUM_FRAC && s.mode != JM_NUM_EXP) { s.mode = JM_NUM_DOT; return true; }
            if ((c == 'e' || c == 'E') && s.mode != JM_NUM_EXP) { s.mode = JM_NUM_E; return true; }
            s.mode = JM_AFTER;         // the number ended: this byte belongs to the ws slot behind it
            s.cnt = 0;
            break;
        default:
            break;
    }
    if (s.mode > JM_AFTER) return false;
    // ---- a ws slot, then what the mode expects ----
    if (c == ' ') {
        if (s.cnt == 0) { s.cnt = JSON_WS_CLOSED; return true; }
        if (s.cnt <= JSON_WS_MAX) { ++s.cnt; return true; }
        return false;
    }
    if (c == '\t') {
        if (s.cnt >= 1 && s.cnt <= JSON_WS_MAX) { ++s.cnt; return true; }
        return false;
    }
    if (c == '\n') {
        if (s.cnt == 0) { s.cnt = 1; return true; }
        return false;
    }
    s.cnt = 0;
    switch (s.mode) {
        case JM_OBJ_FIRST:
            if (c == '}') { json_close(s); return true; }
            if (c == '"') { s.mode = JM_STR; s.key = 1; return true; }
            return false;
        case JM_OBJ_KEY:
            if (c == '"') { s.mode = JM_STR; s.key = 1; return true; }
            return false;
        case JM_COLON:
            if (c == ':') { s.mode = JM_VALUE; return true; }
            return false;
        case JM_VALUE:
            return json_begin_value(s, c);
        case JM_ARR_FIRST:
            if (c == ']') { json_close(s); return true; }
            return json_begin_value(s, c);
        case JM_AFTER:
            if (s.depth == 0) return false;
            if (c == ',') { s.mode = json_top_is_object(s) ? JM_OBJ_KEY : JM_VALUE; return true; }
            if (c == '}' && json_top_is_object(s)) { json_close(s); return true; }
            if (c == ']' && !json_top_is_object(s)) { json_close(s); return true; }
            return false;
        default:
            return false;
    }
}

// the root object has closed: a stop token may end the generation here (anywhere within the trailing ws)
JSON_HD bool json_done(const JsonState& s) { return s.mode == JM_AFTER && s.depth == 0; }

// a run of bytes from s; false as soon as one is refused
JSON_HD bool json_run(JsonState& s, const uint8_t* p, int n) {
    for (int i = 0; i < n; ++i)
        if (!json_step(s, p[i])) return false;
    return true;
}

// per-token class bit (schema_mask.cu): every byte is printable ASCII other than '"' and '\' -- such a token is accepted whole in
// the string-body state without the byte loop
constexpr uint8_t JSON_CLS_PLAIN = 1;

}  // namespace gl
