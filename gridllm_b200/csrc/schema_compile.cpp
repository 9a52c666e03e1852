// JSON schema -> the node table of schema_fsm.h (gl_format_schema; the subset is stated in include/gridllm_native.h).  A small
// JSON parser that keeps the order of object members, then the compiler: it resolves local $refs, orders each object's
// properties (required ones first, then the optional ones, each in `properties` order), spells keys and enum members
// canonically, checks that union alternatives start with disjoint bytes, computes every node's least document depth and writes
// one blob (SchemaHeader, nodes, lists, literal offsets, literal bytes) that the device reads as it is.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "../../include/gridllm_native.h"
#include "schema_fsm.h"

namespace gl {

namespace {

// ---- JSON values ----------------------------------------------------------------------------------------------------------
struct JVal {
    enum Kind { NUL, BOOL, NUM, STR, ARR, OBJ } kind = NUL;
    bool b = false;
    std::string s;                                         // NUM: the text as written; STR: the decoded UTF-8
    std::vector<std::unique_ptr<JVal>> items;
    std::vector<std::pair<std::string, std::unique_ptr<JVal>>> members;
    const JVal* get(const char* k) const {
        for (auto& m : members)
            if (m.first == k) return m.second.get();
        return nullptr;
    }
};

struct Parser {
    const uint8_t* p;
    size_t n, i = 0;
    std::string err;
    void ws() { while (i < n && (p[i] == ' ' || p[i] == '\t' || p[i] == '\n' || p[i] == '\r')) ++i; }
    bool fail(const char* m) { if (err.empty()) err = std::string(m) + " at byte " + std::to_string(i); return false; }
    bool hex4(uint32_t& u) {
        if (i + 4 > n) return fail("truncated \\u escape");
        u = 0;
        for (int k = 0; k < 4; ++k) {
            const uint8_t c = p[i++];
            u <<= 4;
            if (c >= '0' && c <= '9') u |= c - '0';
            else if (c >= 'a' && c <= 'f') u |= c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') u |= c - 'A' + 10;
            else return fail("bad \\u escape");
        }
        return true;
    }
    static void put_utf8(std::string& o, uint32_t u) {
        if (u < 0x80) o += (char)u;
        else if (u < 0x800) { o += (char)(0xC0 | (u >> 6)); o += (char)(0x80 | (u & 0x3F)); }
        else if (u < 0x10000) { o += (char)(0xE0 | (u >> 12)); o += (char)(0x80 | ((u >> 6) & 0x3F)); o += (char)(0x80 | (u & 0x3F)); }
        else {
            o += (char)(0xF0 | (u >> 18)); o += (char)(0x80 | ((u >> 12) & 0x3F));
            o += (char)(0x80 | ((u >> 6) & 0x3F)); o += (char)(0x80 | (u & 0x3F));
        }
    }
    bool string(std::string& o) {
        ++i;                                                  // the opening quote
        JsonState s{};                                        // raw bytes: well-formed UTF-8, no control characters
        s.mode = JM_STR;
        while (true) {
            if (i >= n) return fail("unterminated string");
            const uint8_t c = p[i];
            if (c == '"') { ++i; return true; }
            if (c == '\\') {
                if (++i >= n) return fail("unterminated string");
                const uint8_t e = p[i++];
                switch (e) {
                    case '"': o += '"'; break;
                    case '\\': o += '\\'; break;
                    case '/': o += '/'; break;
                    case 'b': o += '\b'; break;
                    case 'f': o += '\f'; break;
                    case 'n': o += '\n'; break;
                    case 'r': o += '\r'; break;
                    case 't': o += '\t'; break;
                    case 'u': {
                        uint32_t u = 0;
                        if (!hex4(u)) return false;
                        if (u >= 0xDC00 && u <= 0xDFFF) return fail("lone surrogate");
                        if (u >= 0xD800 && u <= 0xDBFF) {
                            uint32_t lo = 0;
                            if (i + 2 > n || p[i] != '\\' || p[i + 1] != 'u') return fail("lone surrogate");
                            i += 2;
                            if (!hex4(lo)) return false;
                            if (lo < 0xDC00 || lo > 0xDFFF) return fail("lone surrogate");
                            u = 0x10000 + ((u - 0xD800) << 10) + (lo - 0xDC00);
                        }
                        put_utf8(o, u);
                        break;
                    }
                    default: return fail("bad escape");
                }
                continue;
            }
            if (!json_step(s, c)) return fail("control character or malformed UTF-8 in a string");
            o += (char)c;
            ++i;
        }
    }
    bool value(JVal& v, int depth) {
        if (depth > 256) return fail("nesting too deep");
        ws();
        if (i >= n) return fail("unexpected end");
        const uint8_t c = p[i];
        if (c == '{') {
            v.kind = JVal::OBJ;
            ++i; ws();
            if (i < n && p[i] == '}') { ++i; return true; }
            while (true) {
                ws();
                if (i >= n || p[i] != '"') return fail("expected a key");
                std::string k;
                if (!string(k)) return false;
                for (auto& m : v.members)
                    if (m.first == k) return fail("duplicate key");
                ws();
                if (i >= n || p[i] != ':') return fail("expected ':'");
                ++i;
                auto child = std::make_unique<JVal>();
                if (!value(*child, depth + 1)) return false;
                v.members.emplace_back(std::move(k), std::move(child));
                ws();
                if (i < n && p[i] == ',') { ++i; continue; }
                if (i < n && p[i] == '}') { ++i; return true; }
                return fail("expected ',' or '}'");
            }
        }
        if (c == '[') {
            v.kind = JVal::ARR;
            ++i; ws();
            if (i < n && p[i] == ']') { ++i; return true; }
            while (true) {
                auto child = std::make_unique<JVal>();
                if (!value(*child, depth + 1)) return false;
                v.items.push_back(std::move(child));
                ws();
                if (i < n && p[i] == ',') { ++i; continue; }
                if (i < n && p[i] == ']') { ++i; return true; }
                return fail("expected ',' or ']'");
            }
        }
        if (c == '"') { v.kind = JVal::STR; return string(v.s); }
        auto word = [&](const char* w) { const size_t l = strlen(w); if (i + l <= n && !memcmp(p + i, w, l)) { i += l; return true; } return false; };
        if (word("true")) { v.kind = JVal::BOOL; v.b = true; return true; }
        if (word("false")) { v.kind = JVal::BOOL; v.b = false; return true; }
        if (word("null")) { v.kind = JVal::NUL; return true; }
        // a number: the JSON automaton checks its syntax
        JsonState s{};
        s.mode = JM_VALUE;
        const size_t a = i;
        while (i < n) {
            const uint8_t d = p[i];
            if (!(d == '-' || d == '+' || d == '.' || d == 'e' || d == 'E' || (d >= '0' && d <= '9'))) break;
            if (!json_step(s, d)) return fail("malformed number");
            ++i;
        }
        if (i == a || !(s.mode == JM_NUM_ZERO || s.mode == JM_NUM_INT || s.mode == JM_NUM_FRAC || s.mode == JM_NUM_EXP))
            return fail("malformed value");
        v.kind = JVal::NUM;
        v.s.assign((const char*)p + a, i - a);
        return true;
    }
};

// Python's json.dumps(s, ensure_ascii=False) of a string, without the quotes
std::string canon_string(const std::string& s) {
    std::string o;
    for (unsigned char c : s) {
        if (c == '"') o += "\\\"";
        else if (c == '\\') o += "\\\\";
        else if (c == '\b') o += "\\b";
        else if (c == '\f') o += "\\f";
        else if (c == '\n') o += "\\n";
        else if (c == '\r') o += "\\r";
        else if (c == '\t') o += "\\t";
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
        else o += (char)c;
    }
    return o;
}

std::string ptr_escape(const std::string& k) {
    std::string o;
    for (char c : k) {
        if (c == '~') o += "~0";
        else if (c == '/') o += "~1";
        else o += c;
    }
    return o;
}

bool is_annotation(const std::string& k) {
    static const char* const A[] = {"title", "description", "$schema", "$id", "$comment", "examples", "default", "deprecated",
                                    "readOnly", "writeOnly", "discriminator"};
    for (const char* a : A)
        if (k == a) return true;
    return false;
}

struct Compiler {
    const JVal* root = nullptr;
    struct Node { SchemaNode n{}; std::vector<uint16_t> list; std::string ptr; };
    std::vector<Node> nodes;
    std::vector<std::string> lits;
    std::map<std::string, int> lit_id;
    std::map<const JVal*, int> memo;
    std::set<const JVal*> resolving;
    int any_node = -1;
    int code = GL_OK;
    std::string err;

    int fail(int c, const std::string& m) { if (code == GL_OK) { code = c; err = m; } return -1; }
    int unsupported(const std::string& m, const std::string& ptr) { return fail(GL_ERR_UNSUPPORTED, m + " at " + (ptr.empty() ? "/" : ptr)); }
    int invalid(const std::string& m, const std::string& ptr) { return fail(GL_ERR_INVALID, m + " at " + (ptr.empty() ? "/" : ptr)); }

    int new_node(uint8_t kind, const std::string& ptr) {
        if ((int)nodes.size() >= SCHEMA_MAX_NODES) return fail(GL_ERR_UNSUPPORTED, "the schema needs more than 4096 nodes");
        Node nd;
        nd.n.kind = kind;
        nd.n.hi = SCHEMA_UNBOUNDED;
        nd.ptr = ptr;
        nodes.push_back(nd);
        return (int)nodes.size() - 1;
    }
    int any() {
        if (any_node < 0) any_node = new_node(SK_ANY, "");
        return any_node;
    }
    int literal(const std::string& s) {
        auto it = lit_id.find(s);
        if (it != lit_id.end()) return it->second;
        if (lits.size() >= 65535) return fail(GL_ERR_UNSUPPORTED, "the schema has more than 65535 literals");
        lits.push_back(s);
        return lit_id[s] = (int)lits.size() - 1;
    }
    // a non-negative integer keyword (<= 65534, the counters' range); -2: absent
    int count(const JVal* s, const char* k, const std::string& ptr) {
        const JVal* v = s->get(k);
        if (!v) return -2;
        if (v->kind != JVal::NUM || v->s.find_first_of(".eE-") != std::string::npos) return invalid(std::string("'") + k + "' must be a non-negative integer", ptr);
        if (v->s.size() > 5 || std::stol(v->s) > 65534) return unsupported(std::string("'") + k + "' above 65534", ptr);
        return (int)std::stol(v->s);
    }
    // the canonical spelling of an enum / const member; "" when it is not a string, integer, boolean or null
    std::string member(const JVal& m) {
        switch (m.kind) {
            case JVal::STR: return "\"" + canon_string(m.s) + "\"";
            case JVal::BOOL: return m.b ? "true" : "false";
            case JVal::NUL: return "null";
            case JVal::NUM:
                if (m.s.find_first_of(".eE") != std::string::npos) return "";
                return m.s == "-0" ? "0" : m.s;
            default: return "";
        }
    }
    static const char* type_of_member(const JVal& m) {
        switch (m.kind) {
            case JVal::STR: return "string";
            case JVal::BOOL: return "boolean";
            case JVal::NUL: return "null";
            default: return "integer";
        }
    }
    const JVal* resolve(const std::string& ref, std::string& ptr) {
        if (ref == "#") { ptr = ""; return root; }
        const char* pre[] = {"#/$defs/", "#/definitions/"};
        for (const char* p : pre) {
            const size_t l = strlen(p);
            if (ref.compare(0, l, p) != 0) continue;
            std::string name, raw = ref.substr(l);
            if (raw.find('/') != std::string::npos) return nullptr;
            for (size_t i = 0; i < raw.size(); ++i) {
                if (raw[i] == '~' && i + 1 < raw.size() && (raw[i + 1] == '0' || raw[i + 1] == '1')) { name += raw[i + 1] == '0' ? '~' : '/'; ++i; }
                else name += raw[i];
            }
            const JVal* defs = root->get(p[2] == '$' ? "$defs" : "definitions");
            if (!defs || defs->kind != JVal::OBJ) return nullptr;
            const JVal* t = defs->get(name.c_str());
            ptr = std::string(p[2] == '$' ? "/$defs/" : "/definitions/") + ptr_escape(name);
            return t;
        }
        return nullptr;
    }

    int compile(const JVal* s, const std::string& ptr) {
        if (code != GL_OK) return -1;
        if (s->kind == JVal::BOOL) {
            if (!s->b) return unsupported("the schema false (no document)", ptr);
            return any();
        }
        if (s->kind != JVal::OBJ) return invalid("a schema must be an object or a boolean", ptr);
        auto it = memo.find(s);
        if (it != memo.end()) return it->second;
        static const char* const KNOWN[] = {"type", "properties", "required", "additionalProperties", "items", "minItems", "maxItems",
                                            "minLength", "maxLength", "enum", "const", "anyOf", "oneOf", "allOf", "$ref", "$defs",
                                            "definitions"};
        std::vector<std::string> used;                       // the keywords that constrain this schema
        for (auto& m : s->members) {
            if (is_annotation(m.first)) continue;
            bool known = false;
            for (const char* k : KNOWN) known = known || m.first == k;
            if (!known) return unsupported("'" + m.first + "' is not supported", ptr);
            if (m.first != "$defs" && m.first != "definitions") used.push_back(m.first);
        }
        auto only = [&](const char* kw, std::initializer_list<const char*> also) -> bool {
            for (auto& u : used) {
                if (u == kw) continue;
                bool ok = false;
                for (const char* a : also) ok = ok || u == a;
                if (!ok) { unsupported("'" + u + "' alongside '" + kw + "' is not supported", ptr); return false; }
            }
            return true;
        };
        if (const JVal* r = s->get("$ref")) {
            if (!only("$ref", {})) return -1;
            std::string tp;
            const JVal* t = r->kind == JVal::STR ? resolve(r->s, tp) : nullptr;
            if (!t) return unsupported("'$ref' " + (r->kind == JVal::STR ? "'" + r->s + "'" : std::string("value")) + " is not a local reference", ptr);
            if (resolving.count(s)) return unsupported("a cycle of '$ref's", ptr);
            resolving.insert(s);
            const int k = compile(t, tp);
            resolving.erase(s);
            return memo[s] = k;
        }
        if (const JVal* a = s->get("allOf")) {
            if (!only("allOf", {})) return -1;
            if (a->kind != JVal::ARR || a->items.size() != 1) return unsupported("'allOf' with other than one member is not supported", ptr);
            if (resolving.count(s)) return unsupported("a cycle of 'allOf's", ptr);
            resolving.insert(s);
            const int k = compile(a->items[0].get(), ptr + "/allOf/0");
            resolving.erase(s);
            return memo[s] = k;
        }
        const JVal* alts = s->get("anyOf");
        const char* akw = "anyOf";
        if (!alts) { alts = s->get("oneOf"); akw = "oneOf"; }
        if (alts) {
            if (!only(akw, {})) return -1;
            if (alts->kind != JVal::ARR || alts->items.empty()) return invalid(std::string("'") + akw + "' must be a non-empty array", ptr);
            const int u = new_node(SK_UNION, ptr);
            if (u < 0) return -1;
            memo[s] = u;
            for (size_t i = 0; i < alts->items.size(); ++i) {
                const int k = compile(alts->items[i].get(), ptr + "/" + akw + "/" + std::to_string(i));
                if (k < 0) return -1;
                nodes[u].list.push_back((uint16_t)k);
            }
            return u;
        }
        // the types this schema allows
        std::vector<std::string> types;
        if (const JVal* t = s->get("type")) {
            if (t->kind == JVal::STR) types.push_back(t->s);
            else if (t->kind == JVal::ARR && !t->items.empty()) {
                for (auto& x : t->items) {
                    if (x->kind != JVal::STR) return invalid("'type' must be a string or an array of strings", ptr);
                    types.push_back(x->s);
                }
            } else return invalid("'type' must be a string or an array of strings", ptr);
            for (auto& x : types)
                if (x != "object" && x != "array" && x != "string" && x != "integer" && x != "number" && x != "boolean" && x != "null")
                    return invalid("unknown type '" + x + "'", ptr);
        }
        const JVal* en = s->get("enum");
        const JVal* cn = s->get("const");
        if (en || cn) {
            if (!only(en ? "enum" : "const", {"type"})) return -1;
            std::vector<const JVal*> ms;
            if (en) {
                if (en->kind != JVal::ARR) return invalid("'enum' must be an array", ptr);
                for (auto& x : en->items) ms.push_back(x.get());
            } else ms.push_back(cn);
            if (ms.empty()) return unsupported("an empty 'enum' (no document)", ptr);
            const int k = new_node(SK_ENUM, ptr);
            if (k < 0) return -1;
            memo[s] = k;
            std::set<std::string> seen;
            for (const JVal* m : ms) {
                const std::string c = member(*m);
                if (c.empty()) return unsupported("an enum member that is not a string, integer, boolean or null", ptr);
                bool typed = types.empty();
                for (auto& t : types) typed = typed || t == type_of_member(*m) || (t == "number" && m->kind == JVal::NUM);
                if (!typed) continue;                            // a member the type rules out is no document
                if (!seen.insert(c).second) continue;
                const int l = literal(c);
                if (l < 0) return -1;
                nodes[k].list.push_back((uint16_t)l);
            }
            if (nodes[k].list.empty()) return unsupported("no 'enum' member matches 'type' (no document)", ptr);
            return k;
        }
        auto has = [&](const char* k) { return s->get(k) != nullptr; };
        if (types.empty()) {                                      // the type the keywords imply
            const bool o = has("properties") || has("required") || has("additionalProperties");
            const bool a = has("items") || has("minItems") || has("maxItems");
            const bool st = has("minLength") || has("maxLength");
            if (o + a + st > 1) return unsupported("keywords of several types without 'type'", ptr);
            if (o) types.push_back("object");
            else if (a) types.push_back("array");
            else if (st) types.push_back("string");
            else return memo[s] = any();
        }
        bool has_num = false;
        for (auto& t : types) has_num = has_num || t == "number";
        std::vector<std::string> ts;                              // integer is part of number
        for (auto& t : types)
            if (!(t == "integer" && has_num) && std::find(ts.begin(), ts.end(), t) == ts.end()) ts.push_back(t);
        int u = -1;
        if (ts.size() > 1) {
            u = new_node(SK_UNION, ptr);
            if (u < 0) return -1;
            memo[s] = u;
        }
        for (auto& t : ts) {
            int k = -1;
            if (t == "object") {
                const JVal* props = s->get("properties");
                const JVal* ap = s->get("additionalProperties");
                const JVal* req = s->get("required");
                if (ap && !(ap->kind == JVal::BOOL && !ap->b))
                    return unsupported("'additionalProperties' other than false is not supported", ptr + "/additionalProperties");
                if (props && props->kind != JVal::OBJ) return invalid("'properties' must be an object", ptr);
                if (req && req->kind != JVal::ARR) return invalid("'required' must be an array", ptr);
                std::vector<std::string> rq;
                if (req)
                    for (auto& x : req->items) {
                        if (x->kind != JVal::STR) return invalid("'required' must hold strings", ptr);
                        if (!props || !props->get(x->s.c_str())) return unsupported("required property '" + x->s + "' is not in 'properties'", ptr + "/required");
                        if (std::find(rq.begin(), rq.end(), x->s) == rq.end()) rq.push_back(x->s);
                    }
                if (!props && !ap) {
                    k = new_node(SK_OBJ_ANY, ptr);
                    if (k < 0) return -1;
                } else {
                    const size_t np = props ? props->members.size() : 0;
                    if (np > (size_t)SCHEMA_MAX_PROPS) return unsupported("more than 255 properties", ptr);
                    k = new_node(SK_OBJ, ptr);
                    if (k < 0) return -1;
                    if (u < 0) memo[s] = k;
                    nodes[k].n.n = (uint16_t)np;
                    nodes[k].n.lo = (uint16_t)rq.size();
                    for (int pass = 0; pass < 2; ++pass)                 // required ones first, then the optional ones
                        for (size_t i = 0; i < np; ++i) {
                            auto& m = props->members[i];
                            const bool r = std::find(rq.begin(), rq.end(), m.first) != rq.end();
                            if (r != (pass == 0)) continue;
                            const int l = literal(canon_string(m.first) + "\"");
                            if (l < 0) return -1;
                            const int vk = compile(m.second.get(), ptr + "/properties/" + ptr_escape(m.first));
                            if (vk < 0) return -1;
                            nodes[k].list.push_back((uint16_t)l);
                            nodes[k].list.push_back((uint16_t)vk);
                        }
                }
            } else if (t == "array") {
                const int lo = count(s, "minItems", ptr), hi = count(s, "maxItems", ptr);
                if (code != GL_OK) return -1;
                if (lo >= 0 && hi >= 0 && lo > hi) return unsupported("'minItems' > 'maxItems' (no document)", ptr);
                k = new_node(SK_ARR, ptr);
                if (k < 0) return -1;
                if (u < 0) memo[s] = k;
                nodes[k].n.lo = (uint16_t)(lo >= 0 ? lo : 0);
                nodes[k].n.hi = (uint16_t)(hi >= 0 ? hi : SCHEMA_UNBOUNDED);
                const JVal* it = s->get("items");
                const int ik = it ? compile(it, ptr + "/items") : any();
                if (ik < 0) return -1;
                nodes[k].n.list = (uint32_t)ik;
            } else if (t == "string") {
                const int lo = count(s, "minLength", ptr), hi = count(s, "maxLength", ptr);
                if (code != GL_OK) return -1;
                if (lo >= 0 && hi >= 0 && lo > hi) return unsupported("'minLength' > 'maxLength' (no document)", ptr);
                k = new_node(SK_STR, ptr);
                if (k < 0) return -1;
                nodes[k].n.lo = (uint16_t)(lo >= 0 ? lo : 0);
                nodes[k].n.hi = (uint16_t)(hi >= 0 ? hi : SCHEMA_UNBOUNDED);
            } else {
                k = new_node(t == "integer" ? SK_INT : t == "number" ? SK_NUM : t == "boolean" ? SK_BOOL : SK_NULL, ptr);
                if (k < 0) return -1;
            }
            if (u >= 0) nodes[u].list.push_back((uint16_t)k);
            else memo[s] = k;
        }
        return u >= 0 ? u : memo[s];
    }

    void first_set(int k, bool out[256]) {
        for (int c = 0; c < 256; ++c) out[c] = false;
        const Node& nd = nodes[k];
        auto on = [&](const char* cs) { for (; *cs; ++cs) out[(uint8_t)*cs] = true; };
        switch (nd.n.kind) {
            case SK_ANY: on("{[\"-0123456789tfn"); break;
            case SK_OBJ_ANY: case SK_OBJ: on("{"); break;
            case SK_ARR: on("["); break;
            case SK_STR: on("\""); break;
            case SK_INT: case SK_NUM: on("-0123456789"); break;
            case SK_BOOL: on("tf"); break;
            case SK_NULL: on("n"); break;
            case SK_ENUM: for (uint16_t l : nd.list) out[(uint8_t)lits[l][0]] = true; break;
            default: break;
        }
    }

    // unions: alternatives that are unions are replaced by theirs, then the alternatives must start with disjoint bytes
    bool finish_unions() {
        for (size_t u = 0; u < nodes.size(); ++u) {
            if (nodes[u].n.kind != SK_UNION) continue;
            std::vector<uint16_t> flat, todo(nodes[u].list.rbegin(), nodes[u].list.rend());
            std::set<int> seen{(int)u};
            while (!todo.empty()) {
                const int k = todo.back();
                todo.pop_back();
                if (nodes[k].n.kind == SK_UNION) {
                    if (!seen.insert(k).second) { unsupported("a union that contains itself", nodes[u].ptr); return false; }
                    todo.insert(todo.end(), nodes[k].list.rbegin(), nodes[k].list.rend());
                } else if (std::find(flat.begin(), flat.end(), k) == flat.end()) flat.push_back((uint16_t)k);
            }
            bool used[256] = {};
            for (uint16_t k : flat) {
                bool f[256];
                first_set(k, f);
                for (int c = 0; c < 256; ++c) {
                    if (f[c] && used[c]) {
                        unsupported("alternatives that can start with the same byte ('" + std::string(1, (char)c) + "') are not supported", nodes[u].ptr);
                        return false;
                    }
                    used[c] = used[c] || f[c];
                }
            }
            nodes[u].list = flat;
        }
        return true;
    }

    // least nesting depth of a document of every node (a fixpoint from "none")
    void depths() {
        for (auto& nd : nodes) nd.n.mind = SCHEMA_INF;
        for (bool changed = true; changed;) {
            changed = false;
            for (auto& nd : nodes) {
                int m = SCHEMA_INF;
                switch (nd.n.kind) {
                    case SK_OBJ_ANY: m = 1; break;
                    case SK_OBJ: {
                        int w = 0;
                        for (int i = 0; i < nd.n.lo; ++i) w = std::max<int>(w, nodes[nd.list[2 * i + 1]].n.mind);
                        m = 1 + w;
                        break;
                    }
                    case SK_ARR: m = 1 + (nd.n.lo > 0 ? nodes[nd.n.list].n.mind : 0); break;
                    case SK_UNION:
                        for (uint16_t k : nd.list) m = std::min<int>(m, nodes[k].n.mind);
                        break;
                    default: m = 0; break;
                }
                if (m > SCHEMA_INF) m = SCHEMA_INF;
                if (m < nd.n.mind) { nd.n.mind = (uint8_t)m; changed = true; }
            }
        }
    }
};

}  // namespace

int schema_compile(const char* text, size_t n, std::vector<uint8_t>& blob, std::string& err) {
    Parser ps{(const uint8_t*)text, n};
    JVal root;
    if (!ps.value(root, 0)) { err = "format schema: malformed JSON: " + ps.err; return GL_ERR_INVALID; }
    ps.ws();
    if (ps.i != n) { err = "format schema: malformed JSON: trailing bytes at byte " + std::to_string(ps.i); return GL_ERR_INVALID; }
    Compiler c;
    c.root = &root;
    const int r = c.compile(&root, "");
    if (c.code == GL_OK) c.finish_unions();
    if (c.code == GL_OK) {
        c.depths();
        const SchemaNode& rn = c.nodes[r].n;
        if (rn.kind != SK_OBJ && rn.kind != SK_OBJ_ANY) c.unsupported("the root must be an object schema", "");
        else if (rn.mind > JSON_MAX_DEPTH) c.unsupported("the smallest document nests deeper than 64", "");
    }
    if (c.code != GL_OK) { err = "format schema: " + c.err; return c.code; }
    // the blob
    std::vector<uint16_t> list;
    for (auto& nd : c.nodes) {
        if (nd.n.kind == SK_OBJ || nd.n.kind == SK_ENUM || nd.n.kind == SK_UNION) {
            nd.n.list = (uint32_t)list.size();
            if (nd.n.kind != SK_OBJ) nd.n.n = (uint16_t)nd.list.size();
            list.insert(list.end(), nd.list.begin(), nd.list.end());
        }
    }
    std::vector<uint32_t> lit_off{0};
    std::string lit;
    for (auto& l : c.lits) { lit += l; lit_off.push_back((uint32_t)lit.size()); }
    SchemaHeader h{};
    h.root = (uint32_t)r;
    h.n_nodes = (uint32_t)c.nodes.size();
    h.n_list = (uint32_t)list.size();
    h.n_lits = (uint32_t)c.lits.size();
    h.off_nodes = sizeof(SchemaHeader);
    h.off_list = h.off_nodes + h.n_nodes * sizeof(SchemaNode);
    h.off_lit_off = (h.off_list + h.n_list * 2 + 3) / 4 * 4;
    h.off_lit = h.off_lit_off + (uint32_t)lit_off.size() * 4;
    blob.assign(h.off_lit + lit.size(), 0);
    memcpy(blob.data(), &h, sizeof h);
    for (size_t i = 0; i < c.nodes.size(); ++i) memcpy(blob.data() + h.off_nodes + i * sizeof(SchemaNode), &c.nodes[i].n, sizeof(SchemaNode));
    if (!list.empty()) memcpy(blob.data() + h.off_list, list.data(), list.size() * 2);
    memcpy(blob.data() + h.off_lit_off, lit_off.data(), lit_off.size() * 4);
    if (!lit.empty()) memcpy(blob.data() + h.off_lit, lit.data(), lit.size());
    return GL_OK;
}

}  // namespace gl
