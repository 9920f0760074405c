// CouchDB's key and value checks in the MVCC stage (fabgpu_state_database(ctx, FABGPU_STATEDB_COUCHDB)): validateWriteset
// (validation/batch_preparer.go:317-330) over ValidateKeyValue (statecouchdb.go:427, couchdoc_conv.go:37-57,278-297), run as a pre-pass
// that turns a VALID transaction into INVALID_WRITESET (24) or 254 before the stage proper reads the flags.  Host+device code: the tests'
// host build runs the same pre-pass one item at a time.
//
// A key is invalid when it is not valid UTF-8 (Go's utf8.ValidString), starts with '_', or is empty.  A value is invalid when Go 1.14's
// json.Unmarshal into a map[string]interface{} succeeds and some top-level member name equals "~version" or starts with '_'.  That is:
// the bytes pass encoding/json's checkValid scanner, the top-level value is an object (null decodes to no fields; any other type is a
// type error), no number anywhere fails strconv.ParseFloat(s, 64) (an overflow is a saved UnmarshalTypeError), and a member name of the
// top object, unescaped, is reserved.  A value of at most CV_SHORT_MAX bytes is scanned by one thread in one pass (cv_short): the
// scanner as a state machine with a bit stack of the open containers, each number's overflow verdict and each top-level name's check
// taken as the scan passes them.  A longer one is scanned by one CTA, tile by tile (cv_long_cta).  Both give the same verdict bits.
#pragma once
#include "stateset.cuh"

namespace fabgpu { namespace bdev {

// Values up to this length take the one-thread scan (cv_short), longer ones one CTA each (cv_long_*)
#define CV_SHORT_MAX 16384u
// Open containers the scan tracks; a deeper value is 254 (Go 1.14's decoder has no nesting limit)
#define CV_DEPTH 128u

// the verdict bits of cv_short and cv_long_cta
enum : uint32_t { CV_SYNTAX_OK = 1, CV_TOP_OBJECT = 2, CV_NUM_ERR = 4, CV_NUM_UNDET = 8, CV_RESERVED = 16, CV_CUT = 32 };
// a write's code: valid, INVALID_WRITESET, undecided
enum : uint8_t { CW_OK = 0, CW_INVALID = 1, CW_UNDET = 2 };
// TxValidationCode INVALID_WRITESET
enum : uint8_t { TXC_INVALID_WRITESET = 24 };

// utf8.ValidString: no overlong forms, surrogates, code points above U+10FFFF or truncated sequences
BD_HD bool cv_utf8(const uint8_t* p, uint32_t n)
{
    for (uint32_t i = 0; i < n;) {
        const uint32_t c = p[i];
        if (c < 0x80) { i++; continue; }
        uint32_t need, lo = 0x80, hi = 0xbf;
        if (c >= 0xc2 && c <= 0xdf) need = 1;
        else if (c >= 0xe0 && c <= 0xef) { need = 2; if (c == 0xe0) lo = 0xa0; else if (c == 0xed) hi = 0x9f; }
        else if (c >= 0xf0 && c <= 0xf4) { need = 3; if (c == 0xf0) lo = 0x90; else if (c == 0xf4) hi = 0x8f; }
        else return false;
        if (n - i <= need) return false;
        if (p[i + 1] < lo || p[i + 1] > hi) return false;
        for (uint32_t k = 2; k <= need; k++) if ((p[i + k] & 0xc0) != 0x80) return false;
        i += need + 1;
    }
    return true;
}

// validateKey: a key CouchDB can hold
BD_HD bool cv_key_ok(const uint8_t* p, uint32_t n) { return n > 0 && p[0] != '_' && cv_utf8(p, n); }

// The least decimal that ParseFloat rounds to +Inf is H = 2^1024 - 2^970 (the midpoint above MaxFloat64 rounds to even, upwards),
// 0.17976931348623158079372897140530341507993... x 10^309.  A number whose first 40 significant digits equal H's, with exponent 309, is
// not decided here.
#define CV_HD 40
BD_HD int cv_h_digit(uint32_t i)
{
    const char* h = "1797693134862315807937289714053034150799";
    return h[i] - '0';
}

struct CvNum { int32_t x; uint32_t nsig, e; int8_t cmp; uint8_t sig, frac, eneg; };

BD_HD void cv_num_digit(CvNum& m, uint32_t d)
{
    if (!m.sig && d == 0) { if (m.frac) m.x--; return; }       // leading zeros: "0" and the zeros after "0."
    m.sig = 1;
    if (!m.frac) m.x++;
    if (m.cmp == 0 && m.nsig < CV_HD) { const int h = cv_h_digit(m.nsig); if ((int)d != h) m.cmp = (int)d < h ? -1 : 1; }
    if (m.nsig < CV_HD) m.nsig++;
}

// 0: ParseFloat succeeds, CV_NUM_ERR: it overflows, CV_NUM_UNDET: not decided.  The value is 0.S x 10^(x + exponent) with S the
// significant digits.  readFloat stops accumulating an exponent once it reaches 10000 (as recalled), so such exponents are not decided.
BD_HD uint32_t cv_num_end(const CvNum& m)
{
    if (!m.sig) return 0;
    if (m.e >= 10000) return CV_NUM_UNDET;
    const int32_t x = m.x + (m.eneg ? -(int32_t)m.e : (int32_t)m.e);
    if (x != 309) return x > 309 ? CV_NUM_ERR : 0;
    if (m.cmp) return m.cmp > 0 ? CV_NUM_ERR : 0;
    return m.nsig >= CV_HD ? CV_NUM_UNDET : 0;                 // fewer digits that match: below H, whose later digits are not all 0
}

enum : uint8_t {
    CS_VALUE, CS_ARR_FIRST, CS_OBJ_FIRST, CS_OBJ_KEY, CS_COLON, CS_AFTER, CS_END,
    CS_STR, CS_ESC, CS_U, CS_LIT,
    CS_N_MINUS, CS_N_ZERO, CS_N_INT, CS_N_DOT, CS_N_FRAC, CS_N_E, CS_N_ESIGN, CS_N_EXP
};

BD_HD bool cv_space(uint32_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n'; }
BD_HD int cv_hex(uint32_t c) { return c >= '0' && c <= '9' ? (int)c - '0' : c >= 'a' && c <= 'f' ? (int)c - 'a' + 10 : c >= 'A' && c <= 'F' ? (int)c - 'A' + 10 : -1; }

// The verdict bits of one value, one thread in one pass.  0: a syntax error; CV_CUT (with CV_TOP_OBJECT when the top-level value is
// an object, and no other bit): a container deeper than CV_DEPTH opens before any syntax error.  The scan reads the value a byte at a
// time, so it is bound by the latency of its loads: values longer than CV_SHORT_MAX take cv_long_* instead.
BD_HD uint32_t cv_short(const uint8_t* p, uint32_t n)
{
    uint32_t stk[CV_DEPTH / 32] = {0, 0, 0, 0};                    // bit d: container d + 1 is an object
    uint32_t depth = 0, out = 0, lit_i = 0, u_n = 0, u_v = 0, name_pos = 0;
    const char* lit = "";
    bool key = false, top_key = false, name_first = false, name_bad = false;
    uint8_t st = CS_VALUE;
    CvNum m{0, 0, 0, 0, 0, 0, 0};
    // one unescaped character of a top-level member name (-1: not ASCII)
    auto name_char = [&](int c) {
        if (name_first && c == '_') out |= CV_RESERVED;
        name_first = false;
        const char* v = "~version";
        if (name_pos < 8 && c == v[name_pos]) name_pos++; else name_bad = true;
    };
    auto in_obj = [&]() { return depth && ((stk[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1u); };
    auto done_value = [&]() { st = depth ? CS_AFTER : CS_END; };
    for (uint32_t i = 0; i <= n; i++) {
        const uint32_t c = i < n ? p[i] : 256u;                    // 256: the end of the input
        if (st >= CS_N_MINUS) {                                    // a number: continue it, or end it and take c afresh
            const bool dig = c >= '0' && c <= '9';
            switch (st) {
            case CS_N_MINUS: if (c == '0') st = CS_N_ZERO; else if (dig) { cv_num_digit(m, c - '0'); st = CS_N_INT; } else return 0; continue;
            case CS_N_ZERO: if (c == '.') { st = CS_N_DOT; m.frac = 1; continue; } if (c == 'e' || c == 'E') { st = CS_N_E; continue; } break;
            case CS_N_INT:
                if (dig) { cv_num_digit(m, c - '0'); continue; }
                if (c == '.') { st = CS_N_DOT; m.frac = 1; continue; }
                if (c == 'e' || c == 'E') { st = CS_N_E; continue; }
                break;
            case CS_N_DOT: if (dig) { cv_num_digit(m, c - '0'); st = CS_N_FRAC; continue; } return 0;
            case CS_N_FRAC:
                if (dig) { cv_num_digit(m, c - '0'); continue; }
                if (c == 'e' || c == 'E') { st = CS_N_E; continue; }
                break;
            case CS_N_E: if (c == '+' || c == '-') { m.eneg = c == '-'; st = CS_N_ESIGN; continue; } if (dig) { m.e = c - '0'; st = CS_N_EXP; continue; } return 0;
            case CS_N_ESIGN: if (dig) { m.e = c - '0'; st = CS_N_EXP; continue; } return 0;
            default: if (dig) { if (m.e < 10000) m.e = m.e * 10 + (c - '0'); continue; } break;
            }
            out |= cv_num_end(m);
            done_value();
        }
        switch (st) {
        case CS_STR:
            if (c == 256u || c < 0x20) return 0;
            if (c == '"') {
                if (top_key && !name_bad && name_pos == 8) out |= CV_RESERVED;
                if (key) st = CS_COLON; else done_value();
                key = top_key = false;
            } else if (c == '\\') st = CS_ESC;
            else if (top_key) name_char(c < 0x80 ? (int)c : -1);
            continue;
        case CS_ESC:
            if (c == 'u') { st = CS_U; u_n = u_v = 0; continue; }
            {
                int e = c == '"' || c == '\\' || c == '/' ? (int)c : c == 'b' ? 8 : c == 'f' ? 12 : c == 'n' ? 10 : c == 'r' ? 13 : c == 't' ? 9 : -2;
                if (e == -2) return 0;
                if (top_key) name_char(e);
            }
            st = CS_STR;
            continue;
        case CS_U: {
            const int h = c < 256u ? cv_hex(c) : -1;
            if (h < 0) return 0;
            u_v = u_v * 16 + h;
            if (++u_n == 4) { if (top_key) name_char(u_v < 0x80 ? (int)u_v : -1); st = CS_STR; }
            continue;
        }
        case CS_LIT:
            if (c != (uint32_t)(uint8_t)lit[lit_i]) return 0;
            if (lit[++lit_i] == 0) done_value();
            continue;
        default: break;
        }
        if (cv_space(c)) continue;
        if (c == 256u) return st == CS_END ? out | CV_SYNTAX_OK : 0;
        switch (st) {
        case CS_END: return 0;
        case CS_COLON: if (c != ':') return 0; st = CS_VALUE; continue;
        case CS_OBJ_FIRST: case CS_OBJ_KEY:
            if (c == '}' && st == CS_OBJ_FIRST) { depth--; done_value(); continue; }
            if (c != '"') return 0;
            st = CS_STR; key = true; top_key = depth == 1;
            name_first = true; name_bad = false; name_pos = 0;
            continue;
        case CS_AFTER:
            if (c == ',') { st = in_obj() ? CS_OBJ_KEY : CS_VALUE; continue; }
            if (c == (in_obj() ? '}' : ']')) { depth--; done_value(); continue; }
            return 0;
        case CS_ARR_FIRST:
            if (c == ']') { depth--; done_value(); continue; }
            break;
        default: break;
        }
        // a value
        if (c == '{' || c == '[') {
            if (depth == 0 && c == '{') out |= CV_TOP_OBJECT;
            if (depth == CV_DEPTH) return (out & CV_TOP_OBJECT) | CV_CUT;
            const uint32_t b = 1u << (depth & 31);
            stk[depth >> 5] = c == '{' ? (stk[depth >> 5] | b) : (stk[depth >> 5] & ~b);
            depth++;
            st = c == '{' ? CS_OBJ_FIRST : CS_ARR_FIRST;
        } else if (c == '"') { st = CS_STR; key = top_key = false; }
        else if (c == '-' || (c >= '0' && c <= '9')) {
            m = CvNum{0, 0, 0, 0, 0, 0, 0};
            if (c == '-') st = CS_N_MINUS;
            else if (c == '0') st = CS_N_ZERO;
            else { cv_num_digit(m, c - '0'); st = CS_N_INT; }
        } else if (c == 't' || c == 'f' || c == 'n') {
            lit = c == 't' ? "true" : c == 'f' ? "false" : "null"; lit_i = 1; st = CS_LIT;
        } else return 0;
    }
    return 0;                                                      // (not reached: the end of the input returns above)
}

// A write's code from the verdict of its value
BD_HD uint8_t cv_code(uint32_t v)
{
    if (v & CV_CUT) return v & CV_TOP_OBJECT ? CW_UNDET : CW_OK;    // the scan stopped: only an object can be invalid
    if (!(v & CV_SYNTAX_OK) || !(v & CV_TOP_OBJECT) || (v & CV_NUM_ERR) || !(v & CV_RESERVED)) return CW_OK;
    return v & CV_NUM_UNDET ? CW_UNDET : CW_INVALID;
}

// ---- the long path: one CTA per value -------------------------------------------------------------------------------------------
// The value goes tile by tile (CV_LT lanes of CV_CH bytes), with state carried between tiles.  Each lane owns its chunk; five CTA scans
// give every lane what the bytes before its chunk leave behind:
//   1. backslash runs (all-backslash flag, trailing run parity) -> whether the chunk's first byte is escaped;
//   2. unescaped quotes (parity, prefix XOR) -> whether the chunk starts inside a string;
//   3. tokens (depth change, last token kind) -> depth and the previous token at the chunk's start;
//   4. openers (per nesting level, the type of the last one) -> the type of every open container (the bit stack at the chunk's start);
//   5. whether the previous token is an object key.
// Then each lane checks what starts in its chunk: string bytes and escapes, each token against the one before it in the grammar of its
// innermost container (object `{` -> key | `}`, key -> `:`, `:` -> value, value -> `,` | `}`, `,` -> key; array `[` -> value | `]`,
// value -> `,` | `]`, `,` -> value; one top-level value), each number or literal (the lane where it starts walks it, as cv_short
// does), and the first characters of each top-level member name.  A syntax error and a container opening past CV_DEPTH are recorded at
// their byte positions; the earlier decides, as in cv_short's left-to-right scan.  No lane reads more than its chunk, plus the token
// that starts in it: a value's bytes cost one lane time only inside one number or literal.
#define CV_LT 256u
enum : uint32_t { CV_LT_THREADS = CV_LT };
#define CV_CH 64u
enum : uint8_t { TK_NONE = 0, TK_OBJ, TK_ARR, TK_COBJ, TK_CARR, TK_COMMA, TK_COLON, TK_STR, TK_SCALAR };

struct CvS1 { uint32_t all, tp; };                     // all bytes backslashes; parity of the trailing backslash run
struct CvS3 { int32_t d; uint32_t lastk; };            // depth change; last token kind
struct CvS4 { uint32_t m[4], b[4]; };                  // levels 1..128 the chunk opens (m) and their types (b: 1 object)
struct CvS5 { uint32_t has, key; };                    // last token of the chunk; whether it is an object key

BD_HD CvS1 cv_op1(CvS1 a, CvS1 b) { CvS1 r; r.all = a.all & b.all; r.tp = b.all ? a.tp ^ b.tp : b.tp; return r; }
BD_HD CvS3 cv_op3(CvS3 a, CvS3 b) { CvS3 r; r.d = a.d + b.d; r.lastk = b.lastk ? b.lastk : a.lastk; return r; }
BD_HD CvS4 cv_op4(CvS4 a, CvS4 b) { CvS4 r; for (int k = 0; k < 4; k++) { r.m[k] = a.m[k] | b.m[k]; r.b[k] = (a.b[k] & ~b.m[k]) | b.b[k]; } return r; }
BD_HD CvS5 cv_op5(CvS5 a, CvS5 b) { return b.has ? b : a; }

// Per lane: the inputs of its chunk (exclusive scan results, carry of earlier tiles included) and its contributions
struct CvLane {
    CvS1 s1; uint32_t q; CvS3 s3; CvS4 s4; CvS5 s5;    // the chunk's own contributions
    uint32_t esc, ins; int32_t depth; uint32_t prevk, prevkey; CvS4 stack;   // the state at the chunk's start
};

// The CTA's state for one value: the carries between tiles and the verdict so far
struct CvLong {
    const uint8_t* p; uint32_t n;
    CvS1 c1; uint32_t c2; CvS3 c3; CvS4 c4; CvS5 c5;
    uint32_t err, cut, bits;
};

BD_HD bool cv_scalar_byte(uint32_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '.' || c == '+' || c == '-'; }
BD_HD uint32_t cv_tok(uint32_t c)
{
    return c == '{' ? TK_OBJ : c == '[' ? TK_ARR : c == '}' ? TK_COBJ : c == ']' ? TK_CARR : c == ',' ? TK_COMMA : c == ':' ? TK_COLON : TK_NONE;
}
BD_HD uint32_t cv_stack_bit(const CvS4& s, int32_t level) { return level >= 1 && level <= (int32_t)CV_DEPTH ? (s.b[(level - 1) >> 5] >> ((level - 1) & 31)) & 1u : 0u; }

// The state before a token, from the token before it (kind, whether it is a key), the innermost container (obj) and the depth
BD_HD uint8_t cv_state(uint32_t prevk, uint32_t prevkey, uint32_t obj, int32_t d)
{
    switch (prevk) {
    case TK_NONE: return CS_VALUE;
    case TK_OBJ: return CS_OBJ_FIRST;
    case TK_ARR: return CS_ARR_FIRST;
    case TK_COLON: return CS_VALUE;
    case TK_COMMA: return obj ? CS_OBJ_KEY : CS_VALUE;
    case TK_STR: if (prevkey) return CS_COLON; return d ? CS_AFTER : CS_END;
    default: return d ? CS_AFTER : CS_END;
    }
}
BD_HD bool cv_allowed(uint8_t s, uint32_t k, uint32_t obj)
{
    const bool value = k == TK_OBJ || k == TK_ARR || k == TK_STR || k == TK_SCALAR;
    switch (s) {
    case CS_COLON: return k == TK_COLON;
    case CS_OBJ_FIRST: return k == TK_STR || k == TK_COBJ;
    case CS_OBJ_KEY: return k == TK_STR;
    case CS_AFTER: return k == TK_COMMA || (k == TK_COBJ && obj) || (k == TK_CARR && !obj);
    case CS_ARR_FIRST: return k == TK_CARR || value;
    case CS_VALUE: return value;
    default: return false;
    }
}

// The value's bytes as the CTA scan reads them: the current tile from its shared-memory copy t (bytes [tb, te)), the rest from p
struct CvBytes {
    const uint8_t* p; const uint8_t* t; uint32_t tb, te;
    BD_HD uint32_t operator[](uint32_t j) const { return j >= tb && j < te ? t[j - tb] : p[j]; }
};

// A number or literal occupying exactly p[a, b): CV_SYNTAX_OK with its number verdict, or 0
BD_HD uint32_t cv_scalar(const CvBytes& p, uint32_t a, uint32_t b)
{
    const char* lit = p[a] == 't' ? "true" : p[a] == 'f' ? "false" : p[a] == 'n' ? "null" : nullptr;
    if (lit) {
        uint32_t k = 0;
        for (; a + k < b && lit[k]; k++) if (p[a + k] != (uint32_t)(uint8_t)lit[k]) return 0;
        return a + k == b && !lit[k] ? CV_SYNTAX_OK : 0;
    }
    CvNum m{0, 0, 0, 0, 0, 0, 0};
    uint32_t i = a;
    auto dig = [&](uint32_t j) { return j < b && p[j] >= '0' && p[j] <= '9'; };
    if (i < b && p[i] == '-') i++;
    if (i < b && p[i] == '0') i++;
    else if (dig(i)) while (dig(i)) cv_num_digit(m, p[i++] - '0');
    else return 0;
    if (i < b && p[i] == '.') {
        i++; m.frac = 1;
        if (!dig(i)) return 0;
        while (dig(i)) cv_num_digit(m, p[i++] - '0');
    }
    if (i < b && (p[i] == 'e' || p[i] == 'E')) {
        i++;
        if (i < b && (p[i] == '+' || p[i] == '-')) { m.eneg = p[i] == '-'; i++; }
        if (!dig(i)) return 0;
        while (dig(i)) { if (m.e < 10000) m.e = m.e * 10 + (p[i] - '0'); i++; }
    }
    return i == b ? CV_SYNTAX_OK | cv_num_end(m) : 0;
}

// Whether the top-level member name whose opening quote is at q is reserved: at most its first nine characters are read
BD_HD bool cv_name_reserved(const CvBytes& p, uint32_t n, uint32_t q)
{
    const char* v = "~version";
    uint32_t pos = 0, nch = 0, i = q + 1;
    while (i < n && nch < 9) {
        int c;
        const uint32_t b = p[i];
        if (b == '"') break;
        if (b == '\\') {
            if (i + 1 >= n) return false;
            const uint32_t e = p[i + 1];
            if (e == 'u') {
                uint32_t u = 0;
                for (uint32_t k = 2; k < 6; k++) { const int h = i + k < n ? cv_hex(p[i + k]) : -1; if (h < 0) return false; u = u * 16 + h; }
                c = u < 0x80 ? (int)u : -1; i += 6;
            } else {
                c = e == '"' || e == '\\' || e == '/' ? (int)e : e == 'b' ? 8 : e == 'f' ? 12 : e == 'n' ? 10 : e == 'r' ? 13 : e == 't' ? 9 : -2;
                if (c == -2) return false;
                i += 2;
            }
        } else { c = b < 0x80 ? (int)b : -1; i++; }
        if (nch == 0 && c == '_') return true;
        if (pos == nch && pos < 8 && c == v[pos]) pos++;
        nch++;
    }
    return i < n && p[i] == '"' && nch == 8 && pos == 8;
}

BD_HD void cv_min(uint32_t* p, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
BD_HD void cv_or(uint32_t* p, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}

// Lane walk over the chunk [c0, c1) of the value, from the lane's start state.  phase 0: backslash runs; 1: quote parity; 2: depth and
// last token; 3: opener levels; 4: keys; 5: the checks.  Tokens are the structural bytes, the opening quote of a string and the first byte
// of a number or literal.
BD_HD void cv_lane(CvLong& v, CvLane& L, uint32_t c0, uint32_t c1, int phase, const CvBytes& p)
{
    const uint32_t n = v.n;
    if (phase == 0) {
        L.s1.all = 1; L.s1.tp = 0;
        for (uint32_t j = c0; j < c1; j++) { if (p[j] == '\\') L.s1.tp ^= 1; else { L.s1.all = 0; L.s1.tp = 0; } }
        return;
    }
    uint32_t esc = L.esc, ins = L.ins, q = 0, prevk = L.prevk, prevkey = L.prevkey;
    int32_t d = L.depth;
    CvS4 st = L.stack;
    L.s3.d = 0; L.s3.lastk = TK_NONE; L.s5.has = 0; L.s5.key = 0;
    for (int k = 0; k < 4; k++) L.s4.m[k] = L.s4.b[k] = 0;
    for (uint32_t j = c0; j < c1; j++) {
        const uint32_t c = p[j];
        const bool escaped = esc != 0;
        esc = c == '\\' ? esc ^ 1u : 0u;
        if (c == '"' && !escaped) q ^= 1;
        if (phase == 1) continue;
        const bool in_str = ins != 0;
        if (c == '"' && !escaped) ins ^= 1;
        uint32_t k = TK_NONE;
        if (in_str) {
            if (phase < 5 || (c == '"' && !escaped)) continue;
            if (c < 0x20) { cv_min(&v.err, j); continue; }
            if (c == '\\' && !escaped) {                          // an escape starts here
                if (j + 1 >= n) { cv_min(&v.err, n); continue; }
                const uint32_t e = p[j + 1];
                if (e == 'u') { for (uint32_t h = 2; h < 6; h++) if (j + h >= n || cv_hex(p[j + h]) < 0) { cv_min(&v.err, j); break; } }
                else if (!(e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't')) cv_min(&v.err, j);
            }
            continue;
        }
        if (c == '"') k = TK_STR;
        else if (cv_space(c)) continue;
        else if (cv_scalar_byte(c)) {
            if (j > 0 && cv_scalar_byte(p[j - 1])) continue;      // inside a number or literal that starts earlier
            k = TK_SCALAR;
        } else {
            k = cv_tok(c);
            if (k == TK_NONE) { if (phase == 5) cv_min(&v.err, j); continue; }
        }
        // a token at j; before it: depth d, previous token prevk (a key: prevkey), innermost container at level d
        const uint32_t obj = cv_stack_bit(st, d);
        const uint8_t s = cv_state(prevk, prevkey, obj, d);
        const uint32_t key = k == TK_STR && (s == CS_OBJ_FIRST || s == CS_OBJ_KEY);
        if (phase == 5) {
            if (!cv_allowed(s, k, obj)) cv_min(&v.err, j);
            if (k == TK_OBJ || k == TK_ARR) {
                if (d + 1 > (int32_t)CV_DEPTH) cv_min(&v.cut, j);
                if (prevk == TK_NONE && k == TK_OBJ) cv_or(&v.bits, CV_TOP_OBJECT);
            } else if (k == TK_SCALAR) {
                uint32_t e = j;
                while (e < n && cv_scalar_byte(p[e])) e++;
                const uint32_t r = cv_scalar(p, j, e);
                if (!r) cv_min(&v.err, j); else cv_or(&v.bits, r & (CV_NUM_ERR | CV_NUM_UNDET));
            } else if (key && d == 1 && cv_name_reserved(p, n, j)) cv_or(&v.bits, CV_RESERVED);
        }
        if (phase == 3 && (k == TK_OBJ || k == TK_ARR) && d >= 0 && d + 1 <= (int32_t)CV_DEPTH) {
            const uint32_t w = (uint32_t)d >> 5, b = 1u << (d & 31);   // level d + 1 is bit d
            L.s4.m[w] |= b;
            L.s4.b[w] = k == TK_OBJ ? (L.s4.b[w] | b) : (L.s4.b[w] & ~b);
        }
        if (k == TK_OBJ || k == TK_ARR) {
            if (d >= 0 && d + 1 <= (int32_t)CV_DEPTH) {           // (d < 0: after a syntax error, or in phase 2's relative walk)
                const uint32_t w = (uint32_t)d >> 5, b = 1u << (d & 31);
                st.m[w] |= b; st.b[w] = k == TK_OBJ ? (st.b[w] | b) : (st.b[w] & ~b);
            }
            d++; L.s3.d++;
        } else if (k == TK_COBJ || k == TK_CARR) { d--; L.s3.d--; }
        prevk = k; prevkey = key;
        L.s3.lastk = k; L.s5.has = 1; L.s5.key = key;
    }
    L.q = q;
}

BD_HD void cv_long_begin(CvLong& v, const uint8_t* p, uint32_t n)
{
    v.p = p; v.n = n;
    v.c1.all = 1; v.c1.tp = 0; v.c2 = 0; v.c3.d = 0; v.c3.lastk = TK_NONE; v.c5.has = 0; v.c5.key = 0;
    for (int k = 0; k < 4; k++) v.c4.m[k] = v.c4.b[k] = 0;
    v.err = v.cut = UINT32_MAX; v.bits = 0;
}

// After the last tile: the end of the input must close the top-level value outside any string
BD_HD uint32_t cv_long_end(CvLong& v)
{
    const uint32_t obj = cv_stack_bit(v.c4, v.c3.d);
    if (v.c2 || cv_state(v.c3.lastk, v.c5.key, obj, v.c3.d) != CS_END) cv_min(&v.err, v.n);
    if (v.err != UINT32_MAX && (v.cut == UINT32_MAX || v.err <= v.cut)) return 0;
    if (v.cut != UINT32_MAX) return (v.bits & CV_TOP_OBJECT) | CV_CUT;
    return v.bits | CV_SYNTAX_OK;
}

// The long path on the host, one lane at a time (the device kernel runs the same phases and scans across the CTA)
inline uint32_t cv_long_host(const uint8_t* p, uint32_t n)
{
    CvLong v;
    cv_long_begin(v, p, n);
    static thread_local CvLane lanes[CV_LT];
    const CvBytes bytes{p, p, 0, 0};
    for (uint32_t base = 0; base < n; base += CV_LT * CV_CH) {
        auto lo = [&](uint32_t t) { return base + t * CV_CH < n ? base + t * CV_CH : n; };
        auto hi = [&](uint32_t t) { return base + (t + 1) * CV_CH < n ? base + (t + 1) * CV_CH : n; };
        for (uint32_t t = 0; t < CV_LT; t++) cv_lane(v, lanes[t], lo(t), hi(t), 0, bytes);
        for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].esc = v.c1.tp; v.c1 = cv_op1(v.c1, lanes[t].s1); }
        for (uint32_t t = 0; t < CV_LT; t++) cv_lane(v, lanes[t], lo(t), hi(t), 1, bytes);
        for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].ins = v.c2; v.c2 ^= lanes[t].q; }
        for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].depth = v.c3.d; lanes[t].prevk = v.c3.lastk; lanes[t].prevkey = 0; lanes[t].stack = v.c4; }
        for (int ph = 2; ph <= 5; ph++) {
            for (uint32_t t = 0; t < CV_LT; t++) cv_lane(v, lanes[t], lo(t), hi(t), ph, bytes);
            if (ph == 2) for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].depth = v.c3.d; lanes[t].prevk = v.c3.lastk; v.c3 = cv_op3(v.c3, lanes[t].s3); }
            if (ph == 3) for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].stack = v.c4; v.c4 = cv_op4(v.c4, lanes[t].s4); }
            if (ph == 4) for (uint32_t t = 0; t < CV_LT; t++) { lanes[t].prevkey = v.c5.key; v.c5 = cv_op5(v.c5, lanes[t].s5); }
        }
    }
    return cv_long_end(v);
}

#if defined(__CUDACC__)
// Exclusive scan of one T per lane across the CTA (CV_LT threads), the carry of earlier tiles in front; the carry then takes the tile's total
template <typename T, typename Op>
__device__ T cv_scan(T* sh, T mine, T& carry, Op op)
{
    const uint32_t t = threadIdx.x;
    sh[t] = mine;
    __syncthreads();
    for (uint32_t d = 1; d < CV_LT; d <<= 1) {
        T x = sh[t];
        if (t >= d) x = op(sh[t - d], x);
        __syncthreads();
        sh[t] = x;
        __syncthreads();
    }
    const T before = t ? op(carry, sh[t - 1]) : carry;
    const T total = sh[CV_LT - 1];
    __syncthreads();
    carry = op(carry, total);
    return before;
}

// The verdict bits of one value, by the whole CTA (CV_LT threads); the result is valid in every thread
__device__ uint32_t cv_long_cta(const uint8_t* p, uint32_t n)
{
    __shared__ CvLong v;
    __shared__ union { CvS1 a[CV_LT]; uint32_t b[CV_LT]; CvS3 c[CV_LT]; CvS4 d[CV_LT]; CvS5 e[CV_LT]; } sh;
    __shared__ uint4 tile[CV_LT * CV_CH / 16];                     // the tile's bytes, loaded once
    const uint32_t t = threadIdx.x;
    if (t == 0) cv_long_begin(v, p, n);
    __syncthreads();
    CvS1 c1 = v.c1; uint32_t c2 = 0; CvS3 c3 = v.c3; CvS4 c4 = v.c4; CvS5 c5 = v.c5;
    CvLane L;
    for (uint32_t base = 0; base < n; base += CV_LT * CV_CH) {
        const uint32_t lo = min(n, base + t * CV_CH), hi = min(n, lo + CV_CH), te = min(n, base + CV_LT * CV_CH);
        __syncthreads();                                           // the previous tile's walks are done with `tile`
        uint8_t* tb = reinterpret_cast<uint8_t*>(tile);
        for (uint32_t j = base + t; j < te; j += CV_LT) tb[j - base] = p[j];
        __syncthreads();
        const CvBytes bytes{p, tb, base, te};
        cv_lane(v, L, lo, hi, 0, bytes);
        L.esc = cv_scan(sh.a, L.s1, c1, [](CvS1 a, CvS1 b) { return cv_op1(a, b); }).tp;
        cv_lane(v, L, lo, hi, 1, bytes);
        L.ins = cv_scan(sh.b, L.q, c2, [](uint32_t a, uint32_t b) { return a ^ b; });
        L.depth = c3.d; L.prevk = c3.lastk; L.prevkey = 0; L.stack = c4;
        cv_lane(v, L, lo, hi, 2, bytes);
        const CvS3 b3 = cv_scan(sh.c, L.s3, c3, [](CvS3 a, CvS3 b) { return cv_op3(a, b); });
        L.depth = b3.d; L.prevk = b3.lastk;
        cv_lane(v, L, lo, hi, 3, bytes);
        L.stack = cv_scan(sh.d, L.s4, c4, [](CvS4 a, CvS4 b) { return cv_op4(a, b); });
        cv_lane(v, L, lo, hi, 4, bytes);
        L.prevkey = cv_scan(sh.e, L.s5, c5, [](CvS5 a, CvS5 b) { return cv_op5(a, b); }).key;
        cv_lane(v, L, lo, hi, 5, bytes);
    }
    __syncthreads();
    if (t == 0) { v.c2 = c2; v.c3 = c3; v.c4 = c4; v.c5 = c5; v.bits = cv_long_end(v); }
    __syncthreads();
    return v.bits;
}
#endif

// ---- the pre-pass over one block ------------------------------------------------------------------------------------------------
// One public KVWrite of a VALID transaction: its key, and its value when the field is present
struct CvWrite { uint32_t tx; Seg key, val; uint32_t has_val; };

struct CvArrays {
    CvWrite* w; uint32_t W_cap;
    uint32_t* first_w; uint32_t* n_w; uint8_t* undet;   // per transaction; undet: a read or range rule gives 254
    uint8_t* code;                                      // per write (CW_*)
    uint32_t* lng;                                      // the writes whose value takes the long path (ctr[1] of them)
    uint32_t* ctr;                                      // [0] writes handed out (> W_cap: overflow, the host grows the arrays and runs again), [1] long values
};

// Reads and ranges under CouchDB: a public read of a key CouchDB cannot hold, a range bound that is not UTF-8 (ReadDocRange's
// encodeForJSON moves it), and an end key served (itr_exhausted false) that CouchDB cannot hold are 254
BD_HD bool cv_range_undet(const uint8_t* base, Seg info)
{
    MvccRange g;
    mv_range_parse(base, info, g);
    if (g.form == RF_BAD) return false;                            // the stage gives it 254
    return !cv_utf8(base + g.start.off, g.start.len) || !cv_utf8(base + g.end.off, g.end.len) ||
           (!g.exhausted && !cv_key_ok(base + g.end.off, g.end.len));
}

// One thread per transaction: the public writes of a VALID transaction whose write set the stage enumerates, and its read / range rule
BD_HD void cv_scan_tx(const uint8_t* base, const TxDev& tx, uint32_t t, uint8_t tv, CvArrays& a)
{
    a.first_w[t] = 0; a.n_w[t] = 0; a.undet[t] = 0;
    if (tv != TXC_VALID || !mv_reached(tx)) return;
    uint32_t n = 0, q = UINT32_MAX;                                // q: UINT32_MAX while counting, else the next write's entry
    bool undet = false;
    auto walk = [&]() {
        return kl_scan_rwset<true>(base, tx.results, [&](Seg, Seg coll, Seg key, uint32_t g, Seg body) {
            if (g == 1 && q == UINT32_MAX) undet = undet || !cv_key_ok(base + key.off, key.len);
            else if (g == 2 && q == UINT32_MAX) undet = undet || cv_range_undet(base, body);
            else if (g == 3) {
                if (q == UINT32_MAX) { n++; return true; }
                // KVWrite{key = 1, is_delete = 2, value = 3}: the last value field wins
                CvWrite& w = a.w[q++];
                w.tx = t; w.key = key; w.val.off = w.val.len = 0; w.has_val = 0;
                Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
                uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
                while (r.next(f, wt, x, b)) if (f == 3 && wt == 2) { w.val = b; w.has_val = 1; }
            }
            (void)coll;
            return true;
        });
    };
    if (!walk()) return;                                           // the stage leaves the block open
    a.undet[t] = undet ? 1 : 0;
    if (n == 0) return;
    const uint32_t b = kl_atomic_add(a.ctr, n);
    if (b + n > a.W_cap || b + n < b) return;
    a.first_w[t] = b; a.n_w[t] = n;
    q = b;
    walk();
}

// One thread per write: its code, or (a value longer than CV_SHORT_MAX) an entry in the long list for cv_long_kernel
BD_HD void cv_check_write(uint32_t i, const uint8_t* base, CvArrays& a)
{
    const CvWrite& w = a.w[i];
    if (!cv_key_ok(base + w.key.off, w.key.len)) { a.code[i] = CW_INVALID; return; }
    if (w.has_val && w.val.len > CV_SHORT_MAX) { a.lng[kl_atomic_add(a.ctr + 1, 1)] = i; return; }
    a.code[i] = w.has_val ? cv_code(cv_short(base + w.val.off, w.val.len)) : CW_OK;
}

// One thread per transaction: a VALID one becomes 24 when a write is invalid (validateWriteset returns on the first failing write, so
// an undecided write before it does not matter), else 254 when a write or a read / range rule is undecided
BD_HD void cv_flag_tx(uint32_t t, const CvArrays& a, uint8_t* tv)
{
    if (tv[t] != TXC_VALID) return;
    bool inv = false, undet = a.undet[t] != 0;
    for (uint32_t q = a.first_w[t]; q < a.first_w[t] + a.n_w[t]; q++) { inv = inv || a.code[q] == CW_INVALID; undet = undet || a.code[q] == CW_UNDET; }
    if (inv) tv[t] = TXC_INVALID_WRITESET;
    else if (undet) tv[t] = TXC_NOT_VALIDATED;
}

// fabgpu_test_couch_values' path: 0 chooses by length as the stage does, 1 forces the one-thread scan, 2 the CTA one
BD_HD bool cv_test_long(int path, uint32_t len) { return path == 2 || (path == 0 && len > CV_SHORT_MAX); }

#if defined(__CUDACC__)
__global__ void __launch_bounds__(64)
cv_scan_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, uint32_t T, const uint8_t* __restrict__ tv, CvArrays a)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) cv_scan_tx(block, txs[t], t, tv[t], a);
}

__global__ void __launch_bounds__(128)
cv_check_kernel(const uint8_t* __restrict__ block, CvArrays a, uint32_t W)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < W) cv_check_write(i, block, a);
}

__global__ void __launch_bounds__(128)
cv_flag_kernel(CvArrays a, uint8_t* __restrict__ tv, uint32_t T)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) cv_flag_tx(t, a, tv);
}

// One CTA per long value, over the long list
__global__ void __launch_bounds__(CV_LT)
cv_long_kernel(const uint8_t* __restrict__ block, CvArrays a)
{
    for (uint32_t k = blockIdx.x; k < a.ctr[1]; k += gridDim.x) {
        const uint32_t i = a.lng[k];
        const uint32_t v = cv_long_cta(block + a.w[i].val.off, a.w[i].val.len);
        if (threadIdx.x == 0) a.code[i] = cv_code(v);
    }
}

// fabgpu_test_couch_values: cv_test_kernel takes the values of the one-thread scan, cv_test_long_kernel (one CTA per value) the others

__global__ void __launch_bounds__(128)
cv_test_kernel(const uint8_t* __restrict__ blob, const uint32_t* __restrict__ off, uint32_t n, int path, uint32_t* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !cv_test_long(path, off[i + 1] - off[i])) out[i] = cv_short(blob + off[i], off[i + 1] - off[i]);
}

__global__ void __launch_bounds__(CV_LT)
cv_test_long_kernel(const uint8_t* __restrict__ blob, const uint32_t* __restrict__ off, uint32_t n, int path, uint32_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        if (!cv_test_long(path, off[i + 1] - off[i])) continue;
        const uint32_t v = cv_long_cta(blob + off[i], off[i + 1] - off[i]);
        if (threadIdx.x == 0) out[i] = v;
    }
}
#endif

} }  // namespace fabgpu::bdev
