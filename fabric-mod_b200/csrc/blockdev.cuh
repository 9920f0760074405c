// Device-side block pre-pass: the same walk, gates and decisions as blockval.cpp / bccsp_host.cpp, written once as
// host+device code so that (a) the GPU runs it with one thread per transaction straight on the block bytes that are in
// HBM anyway (SURVEY.md section 8f ranks 1 and 3: block pre-pass, DER / low-S gates on the device) and (b) tests can run
// the identical code on the CPU-only build box (tests/host_sim/blockdev_host.cpp).
//
// Reference semantics restated here (see blockval.hpp for the full list):
//   ValidateTransaction / checkSignatureFromCreator / validateEndorserTransaction   core/common/validation/msgvalidation.go:26-320
//   KeyLevelValidator signature set        core/common/validation/statebased/validator_keylevel.go:243-259
//   SignatureSetToValidIdentities          common/policies/policy.go:365-402
//   cauthdsl evaluator                     common/cauthdsl/cauthdsl.go:24-92
//   collection / chaincode policy per write core/common/validation/statebased/validator_keylevel.go:86-142, v20.go:105-163
//   UnmarshalECDSASignature / IsLowS       bccsp/utils/ecdsa.go:43-92 (Go encoding/asn1 DER rules)
// No STL, no allocation: everything is offsets into the block buffer and fixed-size records.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define BD_HD __host__ __device__ __forceinline__
#else
#define BD_HD inline
#endif

#include "txidset.cuh"

namespace fabgpu { namespace bdev {

enum : uint8_t {
    TXC_VALID = 0, TXC_BAD_PAYLOAD = 2, TXC_BAD_COMMON_HEADER = 3, TXC_BAD_CREATOR_SIGNATURE = 4, TXC_INVALID_ENDORSER_TRANSACTION = 5,
    TXC_UNSUPPORTED_TX_PAYLOAD = 7, TXC_BAD_PROPOSAL_TXID = 8, TXC_DUPLICATE_TXID = 9, TXC_ENDORSEMENT_POLICY_FAILURE = 10,
    TXC_TARGET_CHAIN_NOT_FOUND = 14, TXC_BAD_HEADER_EXTENSION = 19, TXC_BAD_RESPONSE_PAYLOAD = 21, TXC_BAD_RWSET = 22, TXC_ILLEGAL_WRITESET = 23,
    TXC_INVALID_CHAINCODE = 25, TXC_NOT_VALIDATED = 254, TXC_INVALID_OTHER_REASON = 255,
    // fabric-protos-go peer/transaction.proto: set only by the v1.4 validator (channels without V2_0Validation)
    TXC_EXPIRED_CHAINCODE = 17, TXC_CHAINCODE_VERSION_CONFLICT = 18
};

// Validator of the channel (core/committer/txvalidator/router.go:43): v20/validator.go with the plugin dispatcher (V2_0Validation), or
// v14/validator.go with the builtin v13 VSCC and chaincode definitions from lscc (V1_3 / V1_4_2 / V1_4_3).
#define BD_MODE_V20 0
#define BD_MODE_V13 1
// TxDev::v13_sys: what the invoked chaincode is to the v1.4 validator (v14/vscc_validator.go:407-417)
#define BD_SYS_APP 0            // an application chaincode: the invoked and every written namespace are validated
#define BD_SYS_QUERY 1          // qscc or cscc: only the invoked namespace is validated, without a version check
#define BD_SYS_LSCC 2           // lscc: deploy / upgrade validation, left to the CPU validator (recorded as soon as the header names it)

#define BD_MAX_SIGNERS 64       // distinct verified signers one policy evaluation handles (`used` is a 64-bit mask); more -> CPU validator
#define BD_MAX_NS 4             // namespaces validated per transaction (the invoked chaincode + those it writes to); more -> CPU validator
#define BD_MAX_NS_SEEN 8        // namespaces of one read/write set checked for duplicates; more -> CPU validator
#define BD_MAX_COLL 8           // named private-data collections written per transaction; more -> CPU validator while a collection table is installed
#define BD_MAX_POLICY_DEPTH 12  // deepest node of a policy tree eval_policy walks (root = 0); fabgpu_msp_configure refuses deeper trees
#define BD_ENDS_HINT 16         // job-array sizing: expected endorsements per transaction (the capacity is a parameter, see JobArrays::J_cap)
#define BD_WRITES_HINT 8        // write-record sizing while a key policy table is installed: expected writes per transaction (KlArrays::W_cap)
#define BD_MAX_NEED 16          // distinct policy roots one transaction is checked against; more -> CPU validator
#define KP_UNDECIDABLE (-2)     // key policy table root: the key's validation parameter is not one the device may evaluate
#define KP_REMOVED (-3)         // key policy table slot whose entry was removed (probes continue past it)

struct Seg { uint32_t off, len; };

// ---- MSP view on the device --------------------------------------------------------------------------------------------
struct MspDev {
    const uint8_t* id_blob;       // serialized identities back to back
    const uint32_t* id_off;       // n_ids + 1
    const int32_t* key_slot;      // per identity: big-table slot (>= 0), small-table code (<= -2) or -1
    const uint8_t* valid;         // per identity: identity.Validate()
    const int32_t* msp_code;      // per identity: code of its MSP id (equal ids <=> equal codes)
    const int32_t* group;         // per identity: de-duplication id -- Mspid + certificate (policy.go:380-386): two serializations of one
                                  // certificate share it; null = every table entry is its own group
    const uint8_t* keys_xy;       // per identity: X || Y (64 bytes), for signatures whose key has no table
    const uint64_t* ht_hash;      // open-addressing table, size ht_size (power of two); 0 = empty
    const int32_t* ht_idx;
    uint32_t ht_size;
    int32_t n_ids;
};

// Hash of a serialized identity from 16 + 32 + 32 + 24 sampled bytes.  A SerializedIdentity is the MSP id followed by a PEM certificate: every
// identity of an MSP starts with the same bytes and ends with the same "-----END CERTIFICATE-----" footer, so head and tail alone (round 1) put all
// of an MSP's identities into ONE probe chain -- harmless with a dozen identities, the slowest stage of a block with 2 000 client certificates
// (the creator pass of block_resolve_kernel walked the whole chain per lookup).  The two inner windows fall into the base64
// body: the middle (subject / public key) and the end of the signature just before the footer.
BD_HD uint64_t sample_hash(const uint8_t* p, uint32_t n)
{
    uint64_t h = 1469598103934665603ull ^ n;
    const uint32_t head = n < 16 ? n : 16, tail = n < 24 ? n : 24;
    for (uint32_t i = 0; i < head; i++) h = (h ^ p[i]) * 1099511628211ull;
    if (n >= 160) {
        for (uint32_t i = n / 2 - 16; i < n / 2 + 16; i++) h = (h ^ p[i]) * 1099511628211ull;
        for (uint32_t i = n - 72; i < n - 40; i++) h = (h ^ p[i]) * 1099511628211ull;
    }
    for (uint32_t i = n - tail; i < n; i++) h = (h ^ p[i]) * 1099511628211ull;
    return h ? h : 1;
}

BD_HD bool bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t n)
{
#if defined(__CUDA_ARCH__)
    // ~1 KiB identities are compared four times per transaction: go by aligned 32-bit words on both sides, re-aligning
    // each stream with a funnel shift (reads stay inside the 4-byte-aligned words that contain the ranges).
    if (n >= 8) {
        const uint32_t sa = 8u * (uint32_t)((uintptr_t)a & 3u), sb = 8u * (uint32_t)((uintptr_t)b & 3u);
        const uint32_t* pa = reinterpret_cast<const uint32_t*>((uintptr_t)a & ~(uintptr_t)3);
        const uint32_t* pb = reinterpret_cast<const uint32_t*>((uintptr_t)b & ~(uintptr_t)3);
        const uint32_t words = n >> 2;
        // Eight words per step with no exit in between: the sixteen-plus loads of a step are in flight together (with an
        // exit test after every word each ~1 KiB identity cost ~275 dependent HBM round trips).
        uint32_t k = 0;
        for (; k + 8 <= words; k += 8) {
            uint32_t xa[9], xb[9];
#pragma unroll
            for (int q = 0; q < 9; q++) { xa[q] = pa[k + q]; xb[q] = pb[k + q]; }    // word k+8 lies inside the range or its slack
            uint32_t diff = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) diff |= __funnelshift_r(xa[q], xa[q + 1], sa) ^ __funnelshift_r(xb[q], xb[q + 1], sb);
            if (diff) return false;
        }
        for (; k < words; k++) {
            const uint32_t wa = __funnelshift_r(pa[k], pa[k + 1], sa), wb = __funnelshift_r(pb[k], pb[k + 1], sb);
            if (wa != wb) return false;
        }
        for (uint32_t i = words << 2; i < n; i++) if (a[i] != b[i]) return false;
        return true;
    }
#endif
    for (uint32_t i = 0; i < n; i++) if (a[i] != b[i]) return false;
    return true;
}

BD_HD int32_t msp_find(const MspDev& m, const uint8_t* p, uint32_t n)
{
    if (m.ht_size == 0) return -1;
    const uint64_t h = sample_hash(p, n);
    for (uint32_t probe = 0, pos = (uint32_t)h & (m.ht_size - 1); probe < m.ht_size; probe++, pos = (pos + 1) & (m.ht_size - 1)) {
        const uint64_t k = m.ht_hash[pos];
        if (k == 0) return -1;
        if (k != h) continue;
        const int32_t i = m.ht_idx[pos];
        const uint32_t len = m.id_off[i + 1] - m.id_off[i];
        if (len == n && bytes_equal(m.id_blob + m.id_off[i], p, n)) return i;
    }
    return -1;
}

// ---- protobuf wire reader ------------------------------------------------------------------------------------------------
// The only wire reader of the block path: the walk below and blockval.cpp's split_block both use it.
#define BD_FIELD_TOO_LARGE 0xffffffffu   // reported for every field number >= 2^32-1: no message on the path has such a field
struct Reader {
    const uint8_t* base; uint32_t pos, end; bool ok;
    // At most 10 bytes, and the 10th may only carry bit 63 (0 or 1): any other value overflows 64 bits and is an error, as in
    // golang/protobuf's decodeVarint (`if y < 2`), which proto.Unmarshal uses for tags, lengths and values.
    BD_HD bool varint(uint64_t& v)
    {
        v = 0;
        for (int shift = 0; shift < 63; shift += 7) {
            if (pos >= end) { ok = false; return false; }
            const uint8_t c = base[pos++];
            v |= (uint64_t)(c & 0x7f) << shift;
            if (!(c & 0x80)) return true;
        }
        if (pos >= end || base[pos] > 1) { ok = false; return false; }
        v |= (uint64_t)base[pos++] << 63;
        return true;
    }
    BD_HD bool next(uint32_t& field, uint32_t& wt, uint64_t& val, Seg& bytes)
    {
        if (pos >= end) return false;
        uint64_t key;
        if (!varint(key)) return false;
        // A field number that does not fit 32 bits is an unknown field, as in the reference's decoder.  Truncating it instead
        // would read field 2^32 + 2 as field 2 (a second signature, a second Block.data).
        const uint64_t fno = key >> 3;
        field = fno < BD_FIELD_TOO_LARGE ? (uint32_t)fno : BD_FIELD_TOO_LARGE; wt = (uint32_t)(key & 7);
        if (field == 0) { ok = false; return false; }
        if (wt == 0) return varint(val);
        if (wt == 1) { if (end - pos < 8) { ok = false; return false; } pos += 8; return true; }
        if (wt == 5) { if (end - pos < 4) { ok = false; return false; } pos += 4; return true; }
        if (wt == 2) {
            uint64_t ln;
            if (!varint(ln)) return false;
            if ((uint64_t)(end - pos) < ln) { ok = false; return false; }
            bytes.off = pos; bytes.len = (uint32_t)ln; pos += (uint32_t)ln;
            return true;
        }
        ok = false; return false;
    }
};

// Up to 3 selected length-delimited fields (last occurrence wins) and up to 2 varint fields of one message.
struct Sel { uint32_t f[3]; Seg s[3]; bool present[3]; uint32_t uf[2]; uint64_t uv[2]; };

BD_HD bool parse_sel(const uint8_t* base, Seg msg, Sel& sel)
{
    Reader r; r.base = base; r.pos = msg.off; r.end = msg.off + msg.len; r.ok = true;
    for (int i = 0; i < 3; i++) { sel.s[i].off = 0; sel.s[i].len = 0; sel.present[i] = false; }
    sel.uv[0] = sel.uv[1] = 0;
    uint32_t f, wt; uint64_t v = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, v, b)) {
        bool hit = false;
        for (int i = 0; i < 2 && !hit; i++) if (sel.uf[i] && sel.uf[i] == f) { if (wt != 0) return false; sel.uv[i] = v; hit = true; }
        for (int i = 0; i < 3 && !hit; i++) if (sel.f[i] && sel.f[i] == f) { if (wt != 2) return false; sel.s[i] = b; sel.present[i] = true; hit = true; }
    }
    return r.ok;
}
BD_HD Sel make_sel(uint32_t f0, uint32_t f1 = 0, uint32_t f2 = 0, uint32_t u0 = 0, uint32_t u1 = 0)
{
    Sel s; s.f[0] = f0; s.f[1] = f1; s.f[2] = f2; s.uf[0] = u0; s.uf[1] = u1; return s;
}

// ---- DER gate (Go encoding/asn1 rules; bccsp/utils/ecdsa.go:43-92, bccsp/sw/ecdsa.go:42-54) -----------------------------
// Returns true when every gate passes (r, s written as 32 big-endian bytes).  false covers unmarshal errors, R <= 0,
// S <= 0, high S and r >= 2^256: at block level all of those make identity.Verify fail alike.
BD_HD bool der_tag_len(const uint8_t* b, uint32_t n, uint32_t& off, uint32_t& cls, bool& compound, uint32_t& tag, uint32_t& length)
{
    if (off >= n) return false;
    uint8_t c = b[off++];
    cls = c >> 6; compound = (c & 0x20) != 0; tag = c & 0x1f;
    if (tag == 0x1f) {
        uint64_t t = 0; int shifted = 0;
        for (;;) {
            if (off >= n || shifted == 5) return false;
            c = b[off++];
            if (shifted == 0 && c == 0x80) return false;
            t = (t << 7) | (c & 0x7f); shifted++;
            if (!(c & 0x80)) break;
        }
        if (t > 0x7fffffffull || t < 0x1f) return false;
        tag = (uint32_t)t;
    }
    if (off >= n) return false;
    c = b[off++];
    if (!(c & 0x80)) { length = c & 0x7f; return true; }
    const int nb = c & 0x7f;
    if (nb == 0) return false;
    uint32_t L = 0;
    for (int i = 0; i < nb; i++) {
        if (off >= n) return false;
        c = b[off++];
        if (L >= (1u << 23)) return false;
        L = (L << 8) | c;
        if (L == 0) return false;
    }
    if (L < 0x80) return false;
    length = L;
    return true;
}

BD_HD bool der_int(const uint8_t* b, uint32_t n, uint32_t& off, uint32_t& vo, uint32_t& vl)
{
    if (off == n) return false;
    uint32_t cls, tag, len; bool compound;
    if (!der_tag_len(b, n, off, cls, compound, tag, len)) return false;
    if ((uint64_t)off + len > n) return false;
    if (cls != 0 || tag != 2 || compound || len == 0) return false;
    const uint8_t* p = b + off;
    if (len > 1 && ((p[0] == 0 && !(p[1] & 0x80)) || (p[0] == 0xff && (p[1] & 0x80)))) return false;
    vo = off; vl = len; off += len;
    return true;
}

// Gate outcome as the status code of include/fabgpu_ecdsa.h: 0 = every gate passed (ask the curve arithmetic),
// 1 = (false, nil) because r >= 2^256, 5 = unmarshal error, 6 / 7 = R / S not positive, 8 = high S.
// Order of checks as in bccsp/sw/ecdsa.go:41-54: unmarshal, R > 0, S > 0, then low-S, then ecdsa.Verify's range checks.
BD_HD int gate_signature_status(const uint8_t* sig, uint32_t n, uint8_t* r32, uint8_t* s32)
{
    const uint8_t half[32] = {0x7F, 0xFF, 0xFF, 0xFF, 0x80, 0x00, 0x00, 0x00, 0x7F, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF,
                              0xDE, 0x73, 0x7D, 0x56, 0xD3, 0x8B, 0xCF, 0x42, 0x79, 0xDC, 0xE5, 0x61, 0x7E, 0x31, 0x92, 0xA8};
    if (n == 0) return 5;
    uint32_t off = 0, cls, tag, len; bool compound;
    if (!der_tag_len(sig, n, off, cls, compound, tag, len)) return 5;
    if ((uint64_t)off + len > n) return 5;
    if (cls != 0 || tag != 16 || !compound) return 5;
    const uint8_t* inner = sig + off;
    uint32_t io = 0, ro, rl, so, sl;
    if (!der_int(inner, len, io, ro, rl)) return 5;
    if (!der_int(inner, len, io, so, sl)) return 5;
    const uint8_t* rp = inner + ro; const uint8_t* sp = inner + so;
    const bool r_neg = (rp[0] & 0x80) != 0, s_neg = (sp[0] & 0x80) != 0;
    while (rl > 0 && *rp == 0) { rp++; rl--; }
    while (sl > 0 && *sp == 0) { sp++; sl--; }
    if (r_neg || rl == 0) return 6;                               // R must be larger than zero
    if (s_neg || sl == 0) return 7;                               // S must be larger than zero
    if (sl > 32) return 8;                                        // s >= 2^256 > N/2
    for (int i = 0; i < 32; i++) s32[i] = 0;
    for (uint32_t i = 0; i < sl; i++) s32[32 - sl + i] = sp[i];
    for (int i = 0; i < 32; i++) {                                // s <= N >> 1
        if (s32[i] < half[i]) break;
        if (s32[i] > half[i]) return 8;
    }
    if (rl > 32) return 1;                                        // r >= 2^256 can never be < N: (false, nil)
    for (int i = 0; i < 32; i++) r32[i] = 0;
    for (uint32_t i = 0; i < rl; i++) r32[32 - rl + i] = rp[i];
    return 0;
}

BD_HD bool gate_signature(const uint8_t* sig, uint32_t n, uint8_t* r32, uint8_t* s32)
{
    return gate_signature_status(sig, n, r32, s32) == 0;
}

// ---- per-transaction plan --------------------------------------------------------------------------------------------------
struct ShaJobD { uint32_t off[3]; uint32_t len[3]; };

struct TxDev {
    uint8_t early;                 // decided by structure alone, else TXC_NOT_VALIDATED
    uint8_t htype;
    uint8_t endorser_parse_ok, channel_ok, endorsements_parse_ok, overflow;
    uint8_t disp;                  // plugin dispatcher's structural verdict (dispatcher.go:102-179): TXC_VALID or the code it returns
    uint8_t n_ns;                  // namespaces to validate: wr_ns[0] = the invoked chaincode, then the others it writes to
    int32_t creator_identity;      // -1 unknown
    int32_t creator_has_job;       // creator job index is the transaction index when 1
    Seg txid_ascii;
    Seg phash_claimed;
    uint32_t first_end_job;        // endorsement jobs [first_end_job, first_end_job + n_end_jobs), in endorsement order
    uint32_t n_end_jobs;           // (endorsements without signature bytes get none: they can never verify)
    Seg wr_ns[BD_MAX_NS];
    uint8_t n_coll;                // written collections in coll[]; BD_MAX_COLL + 1 = more than that
    uint8_t pub_ns;                // bit i: wr_ns[i] has public writes, or writes to a collection without a name
    uint8_t coll_ns[BD_MAX_COLL];  // wr_ns index of each written collection's namespace
    Seg coll[BD_MAX_COLL];         // collection_name of each CollectionHashedReadWriteSet with hashed writes or metadata writes
    Seg results;                   // ChaincodeAction.results (the TxReadWriteSet), once dispatch_plan has read it
    uint32_t first_w, n_w;         // write records [first_w, first_w + n_w) of KlArrays::w (key policy table installed only)
    uint8_t kl_bad;                // a write inside the read/write set does not parse: the key-level checks cannot be made here
    uint8_t v13_sys;               // v1.3 mode: BD_SYS_* of the invoked chaincode
    Seg r_ver;                     // ChaincodeAction.chaincode_id.version, once dispatch_plan has read it
};

// One write of a transaction as baseEvaluator.Evaluate walks them (validator_keylevel.go:86-142): a public write, public metadata write,
// hashed write or hashed metadata write.  coll is empty for public keys; key is the key hash for collection keys.
struct WriteRec {
    Seg ns, coll, key;
    uint32_t tx;
    uint32_t slot;                 // metadata-write set entry of the key, 0xffffffff = none (set by the walk for metadata records, by
                                   // the decide stage for the others)
    uint8_t ns_idx;                // TxDev::wr_ns index of the namespace
    uint8_t md;                    // a metadata write
    uint8_t gone;                  // from a transaction that never reaches VSCC (only its metadata writes are recorded)
    uint8_t alias;                 // the entry's first writer has another key with the same hash: its dependency is not decided here
};

// Key-level validation state of one block, used only while a key policy table is installed (w = null: off).  The metadata-write set is
// an open-addressing table of md_size slots keyed by kl_key_hash (0 = empty).  Per entry: md_min, the earliest metadata record
// ((tx << 32) | record index, all ones = none), and md_sum, the VSCC results of its writers so far, which the resolve stage fills in
// index order (KL_SUM_*).  Keys with one hash share an entry; the decide stage marks that (KL_SUM_MIXED, WriteRec::alias) and such a
// dependency is not decided here.
#define KL_SUM_NIL 1u              // a writer with a nil result
#define KL_SUM_UNDET 2u            // a writer whose result is not determined by the block
#define KL_SUM_MIXED 4u            // metadata writers of more than one key
#define KL_SUM_ANY 8u              // some writer
struct KlArrays {
    WriteRec* w = nullptr; uint32_t W_cap = 0;
    uint32_t* counter = nullptr;   // [0]: records handed out (> W_cap: overflow), [1]: nonzero = the block's dependencies cannot be trusted
    uint64_t* md_hash = nullptr; unsigned long long* md_min = nullptr; uint32_t* md_sum = nullptr; uint32_t md_size = 0;
    uint8_t* conflicted = nullptr; // per transaction: bit 0 = an earlier transaction metadata-wrote a key it writes, bit 1 = it metadata-writes
    uint32_t* clist = nullptr;     // scratch of the resolve stage: the marked transactions in index order
};

// Everything plan_tx writes for one transaction besides TxDev: job records live in caller-provided arrays.
struct JobArrays {
    KlArrays kl;                   // write records and the metadata-write set; all null without a key policy table
    ShaJobD* sha;                  // [J_cap + 2 T]: signature messages, then (txid, proposal hash) per transaction
    uint8_t* r; uint8_t* s;        // [J_cap x 32]
    int32_t* key_slot;             // [J_cap]
    int32_t* identity;             // [J_cap]
    uint8_t* qx; uint8_t* qy;      // [J_cap x 32] or null: filled only for keys without a table (generic kernel)
    uint8_t* gate_ok;              // [J_cap]
    uint32_t J_cap;                // capacity; creator jobs occupy [0, T), endorsement jobs [T, T + n_end)
    uint32_t T;
    uint8_t mode = BD_MODE_V20;    // the channel's validator: the dispatcher's codes differ (dispatch_plan)
};

// What the walk leaves for one signature; identity lookup and DER gate are done per job by resolve_job (four times
// more threads than transactions: the walk alone exposed too little parallelism -- ncu: 2 warps/SM, issue active 3 %).
struct RawJob { Seg ident; Seg sig; uint32_t tx; int32_t k; };   // k = -1: creator signature, else endorsement index; tx = 0xffffffff: unused slot

// Wire scan of one message: known fields must carry their wire type (Go's proto.Unmarshal fails otherwise); on_bytes(field, seg)
// is called for every length-delimited KNOWN field in order.  bytes_mask / varint_mask: bit f = field f is known with that type.
template <typename F>
BD_HD bool scan_msg(const uint8_t* base, Seg msg, uint32_t bytes_mask, uint32_t varint_mask, F on_bytes)
{
    Reader r; r.base = base; r.pos = msg.off; r.end = msg.off + msg.len; r.ok = true;
    uint32_t f, wt; uint64_t v = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, v, b)) {
        if (f < 32 && ((bytes_mask >> f) & 1u)) { if (wt != 2) return false; on_bytes(f, b); }
        else if (f < 32 && ((varint_mask >> f) & 1u)) { if (wt != 0) return false; }
    }
    return r.ok;
}
#define BD_F(n) (1u << (n))

BD_HD bool seg_equal(const uint8_t* base, Seg a, Seg b)
{
    if (a.len != b.len) return false;
    for (uint32_t i = 0; i < a.len; i++) if (base[a.off + i] != base[b.off + i]) return false;
    return true;
}

// the four-letter system chaincode names of v14/vscc_validator.go:407-417
BD_HD bool seg_is(const uint8_t* base, Seg a, const char* name)
{
    if (a.len != 4) return false;
    for (uint32_t i = 0; i < 4; i++) if (base[a.off + i] != (uint8_t)name[i]) return false;
    return true;
}

// The plugin dispatcher's structural checks (plugindispatcher/dispatcher.go:102-179), in its order.  chdr_ext: ChannelHeader.extension;
// prp / prp_ext: ProposalResponsePayload bytes and its extension (peer.ChaincodeAction).  Fills tx.disp, tx.wr_ns, tx.n_ns, and
// for the collection policies (validator_keylevel.go:86-142) tx.pub_ns and the written collections tx.coll / tx.coll_ns / tx.n_coll.
// mode BD_MODE_V13: the same walk with the v1.4 validator's codes (v14/vscc_validator.go:69-270): 255 for the chaincode-name and
// version checks, its system-chaincode rules, and tx.v13_sys.
BD_HD void dispatch_plan(const uint8_t* base, Seg chdr_ext, bool has_prp, bool has_prp_ext, Seg prp_ext, TxDev& tx, uint8_t mode = BD_MODE_V20)
{
    tx.disp = TXC_VALID; tx.n_ns = 0; tx.n_coll = 0; tx.pub_ns = 0; tx.v13_sys = BD_SYS_APP;
    // hdrExt = ChaincodeHeaderExtension{chaincode_id = 2}, its ChaincodeID{path = 1, name = 2, version = 3} parsed with it
    Seg h_ccid; h_ccid.off = h_ccid.len = 0; bool has_h_ccid = false;
    if (!scan_msg(base, chdr_ext, BD_F(2), 0, [&](uint32_t, Seg b) { h_ccid = b; has_h_ccid = true; })) { tx.disp = TXC_BAD_HEADER_EXTENSION; return; }
    Seg h_name; h_name.off = h_name.len = 0;
    if (has_h_ccid && !scan_msg(base, h_ccid, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg b) { if (f == 2) h_name = b; })) { tx.disp = TXC_BAD_HEADER_EXTENSION; return; }
    // v1.3 mode: an lscc invocation, before any later check -- whatever stops it at 254 (lscc_mark), the reference may accept the upgrade
    if (mode == BD_MODE_V13 && seg_is(base, h_name, "lscc")) tx.v13_sys = BD_SYS_LSCC;
    // respPayload = GetActionFromEnvelope: ChaincodeAction{results = 1, events = 2, response = 3, chaincode_id = 4}
    if (!has_prp || !has_prp_ext) { tx.disp = TXC_BAD_RESPONSE_PAYLOAD; return; }
    Seg results, events, r_ccid; results.off = results.len = events.off = events.len = r_ccid.off = r_ccid.len = 0;
    bool has_events = false, has_r_ccid = false;
    if (!scan_msg(base, prp_ext, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t f, Seg b) {
            if (f == 1) results = b; else if (f == 2) { events = b; has_events = true; } else if (f == 4) { r_ccid = b; has_r_ccid = true; } })) {
        tx.disp = TXC_BAD_RESPONSE_PAYLOAD; return;
    }
    tx.results = results;
    Seg r_name, r_ver; r_name.off = r_name.len = r_ver.off = r_ver.len = 0;
    if (has_r_ccid && !scan_msg(base, r_ccid, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg b) { if (f == 2) r_name = b; else if (f == 3) r_ver = b; })) {
        tx.disp = TXC_BAD_RESPONSE_PAYLOAD; return;
    }
    tx.r_ver = r_ver;
    // txRWSet.FromProtoBytes(results): TxReadWriteSet{data_model = 1, ns_rwset = 2}, every namespace with its KVRWSet and hashed collections
    Seg seen[BD_MAX_NS_SEEN]; bool wrote[BD_MAX_NS_SEEN], pub[BD_MAX_NS_SEEN]; uint32_t n_seen = 0; bool too_many = false, rw_ok = true;
    const bool top_ok = scan_msg(base, results, BD_F(2), BD_F(1), [&](uint32_t, Seg nsb) {
        if (!rw_ok) return;
        Seg name, kv; name.off = name.len = kv.off = kv.len = 0;
        bool writes = false, pub_w = false;
        // NsReadWriteSet{namespace = 1, rwset = 2, collection_hashed_rwset = 3}
        if (!scan_msg(base, nsb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg b) {
                if (f == 1) name = b; else if (f == 2) kv = b;
                else {                                                  // CollectionHashedReadWriteSet{collection_name = 1, hashed_rwset = 2, pvt_rwset_hash = 3}
                    Seg hashed, cname; hashed.off = hashed.len = cname.off = cname.len = 0;
                    if (!scan_msg(base, b, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg c) { if (g == 1) cname = c; else if (g == 2) hashed = c; })) { rw_ok = false; return; }
                    // HashedRWSet{hashed_reads = 1, hashed_writes = 2, metadata_writes = 3}
                    bool cw = false;
                    if (!scan_msg(base, hashed, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg) { if (g == 2 || g == 3) cw = true; })) rw_ok = false;
                    if (!cw) return;
                    writes = true;
                    // no name: the chaincode policy (v20.go:105-106); otherwise recorded against the namespace's index in seen[]
                    if (cname.len == 0) pub_w = true;
                    else if (tx.n_coll < BD_MAX_COLL) { tx.coll[tx.n_coll] = cname; tx.coll_ns[tx.n_coll] = (uint8_t)n_seen; tx.n_coll++; }
                    else tx.n_coll = BD_MAX_COLL + 1;
                } })) { rw_ok = false; return; }
        if (!rw_ok) return;
        // KVRWSet{reads = 1, range_queries_info = 2, writes = 3, metadata_writes = 4}
        if (!scan_msg(base, kv, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t g, Seg) { if (g == 3 || g == 4) writes = pub_w = true; })) { rw_ok = false; return; }
        if (n_seen < BD_MAX_NS_SEEN) { seen[n_seen] = name; wrote[n_seen] = writes; pub[n_seen] = pub_w; n_seen++; } else too_many = true;
    });
    if (!top_ok || !rw_ok) { tx.disp = TXC_BAD_RWSET; return; }
    if (!has_h_ccid || !has_r_ccid) { tx.disp = TXC_INVALID_OTHER_REASON; return; }
    if (h_name.len == 0 || !seg_equal(base, h_name, r_name) || r_ver.len == 0) { tx.disp = mode == BD_MODE_V13 ? TXC_INVALID_OTHER_REASON : TXC_INVALID_CHAINCODE; return; }
    if (has_events) {                                                  // ChaincodeEvent{chaincode_id = 1 (string), tx_id = 2, event_name = 3, payload = 4}
        Seg ev_cc; ev_cc.off = ev_cc.len = 0;
        if (!scan_msg(base, events, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t f, Seg b) { if (f == 1) ev_cc = b; }) || !seg_equal(base, ev_cc, h_name)) {
            tx.disp = TXC_INVALID_OTHER_REASON; return;
        }
    }
    if (too_many) { tx.disp = TXC_NOT_VALIDATED; return; }              // more namespaces than the device tracks: CPU validator
    tx.wr_ns[0] = h_name; tx.n_ns = 1;
    for (uint32_t i = 0; i < n_seen; i++) {
        for (uint32_t j = 0; j < i; j++) if (seg_equal(base, seen[i], seen[j])) { tx.disp = TXC_ILLEGAL_WRITESET; return; }
    }
    if (mode == BD_MODE_V13) {                                        // v14/vscc_validator.go:151-160,176-190,230-238
        bool w_lscc = false, w_sys = false;
        for (uint32_t i = 0; i < n_seen; i++) {
            if (!wrote[i]) continue;
            w_lscc = w_lscc || seg_is(base, seen[i], "lscc");
            w_sys = w_sys || seg_is(base, seen[i], "vscc") || seg_is(base, seen[i], "escc") || seg_is(base, seen[i], "cscc");
        }
        if (seg_is(base, h_name, "vscc") || seg_is(base, h_name, "escc")) { tx.disp = TXC_ILLEGAL_WRITESET; return; }
        if (tx.v13_sys == BD_SYS_LSCC) { tx.disp = TXC_NOT_VALIDATED; return; }
        if (seg_is(base, h_name, "qscc") || seg_is(base, h_name, "cscc")) {
            tx.v13_sys = BD_SYS_QUERY; tx.wr_ns[0] = h_name; tx.n_ns = 1; tx.n_coll = 0; return;
        }
        if (w_lscc || w_sys) { tx.disp = TXC_ILLEGAL_WRITESET; return; }
    }
    uint8_t wr_of[BD_MAX_NS_SEEN];                                     // seen[] index -> wr_ns index, for the namespaces that wrote
    for (uint32_t i = 0; i < n_seen; i++) {
        if (!wrote[i]) continue;
        if (seg_equal(base, seen[i], h_name)) { wr_of[i] = 0; if (pub[i]) tx.pub_ns |= 1; continue; }
        if (tx.n_ns >= BD_MAX_NS) { tx.disp = TXC_NOT_VALIDATED; return; }
        if (pub[i]) tx.pub_ns |= (uint8_t)(1u << tx.n_ns);
        wr_of[i] = tx.n_ns;
        tx.wr_ns[tx.n_ns++] = seen[i];
    }
    for (uint32_t c = 0; c < tx.n_coll && c < BD_MAX_COLL; c++) tx.coll_ns[c] = wr_of[tx.coll_ns[c]];   // a collection write makes its namespace write
}

// ---- key-level validation parameters: write records and in-block dependencies --------------------------------------------
// FNV-1a over (namespace, collection, key), each with its length: the key policy table's and the metadata-write set's hash.
BD_HD uint64_t kl_key_hash(const uint8_t* ns, uint32_t ns_len, const uint8_t* coll, uint32_t coll_len, const uint8_t* key, uint32_t key_len)
{
    uint64_t h = 1469598103934665603ull ^ ns_len;
    for (uint32_t i = 0; i < ns_len; i++) h = (h ^ ns[i]) * 1099511628211ull;
    h = (h ^ coll_len) * 1099511628211ull;
    for (uint32_t i = 0; i < coll_len; i++) h = (h ^ coll[i]) * 1099511628211ull;
    h = (h ^ key_len) * 1099511628211ull;
    for (uint32_t i = 0; i < key_len; i++) h = (h ^ key[i]) * 1099511628211ull;
    return h ? h : 1;
}
BD_HD uint64_t kl_rec_hash(const uint8_t* base, const WriteRec& w)
{
    return kl_key_hash(base + w.ns.off, w.ns.len, base + w.coll.off, w.coll.len, base + w.key.off, w.key.len);
}
BD_HD bool kl_same_key(const uint8_t* base, const WriteRec& a, const WriteRec& b)
{
    return seg_equal(base, a.ns, b.ns) && seg_equal(base, a.coll, b.coll) && seg_equal(base, a.key, b.key);
}

BD_HD uint32_t kl_atomic_add(uint32_t* p, uint32_t n)
{
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, n);
#else
    const uint32_t b = *p; *p += n; return b;
#endif
}

// Every write of a TxReadWriteSet as rwset.FromProtoBytes reads it, in baseEvaluator.Evaluate's terms (validator_keylevel.go:86-142):
// on_write(namespace, collection, key, is_metadata) for each KVWrite{key = 1} and KVMetadataWrite{key = 1} of a namespace's KVRWSet and each
// KVWriteHash{key_hash = 1} and KVMetadataWriteHash{key_hash = 1} of its collections.  false when a level does not parse.
// Reads (the MVCC stage, stateset.cuh): on_write(namespace, collection, key, field, record) -> bool for every record instead, reads and
// range queries included -- field 1-4 of KVRWSet, 11-13 for field 1-3 of HashedRWSet; a range query has no key; false = does not parse.
template <bool Reads = false, typename F>
BD_HD bool kl_scan_rwset(const uint8_t* base, Seg results, F on_write)
{
    bool ok = true;
    const bool top = scan_msg(base, results, BD_F(2), BD_F(1), [&](uint32_t, Seg nsb) {
        if (!ok) return;
        Seg name, kv; name.off = name.len = kv.off = kv.len = 0;          // NsReadWriteSet{namespace = 1, rwset = 2, collection_hashed_rwset = 3}
        if (!scan_msg(base, nsb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg b) { if (f == 1) name = b; else if (f == 2) kv = b; })) { ok = false; return; }
        // KVRWSet{reads = 1, range_queries_info = 2, writes = 3, metadata_writes = 4}; KVWrite{key = 1, is_delete = 2, value = 3},
        // KVMetadataWrite{key = 1, entries = 2}
        Seg none; none.off = none.len = 0;
        if (!scan_msg(base, kv, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t g, Seg w) {
                if (!ok || (!Reads && g != 3 && g != 4)) return;
                Seg key; key.off = key.len = 0;
                // KVRead{key = 1, version = 2} (Reads); a RangeQueryInfo is handed over unparsed
                if ((!Reads || g != 2) &&
                    !scan_msg(base, w, g == 3 ? BD_F(1) | BD_F(3) : BD_F(1) | BD_F(2), g == 3 ? BD_F(2) : 0, [&](uint32_t h, Seg k) { if (h == 1) key = k; })) { ok = false; return; }
                if constexpr (Reads) { if (!on_write(name, none, key, g, w)) ok = false; }
                else on_write(name, none, key, g == 4);
            })) ok = false;
        if (!ok) return;
        scan_msg(base, nsb, BD_F(3), 0, [&](uint32_t, Seg cb) {          // CollectionHashedReadWriteSet{collection_name = 1, hashed_rwset = 2, pvt_rwset_hash = 3}
            if (!ok) return;
            Seg cname, hashed; cname.off = cname.len = hashed.off = hashed.len = 0;
            if (!scan_msg(base, cb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg c) { if (g == 1) cname = c; else if (g == 2) hashed = c; })) { ok = false; return; }
            // HashedRWSet{hashed_reads = 1, hashed_writes = 2, metadata_writes = 3}; KVWriteHash{key_hash = 1, is_delete = 2, value_hash = 3,
            // is_purge = 4}, KVMetadataWriteHash{key_hash = 1, entries = 2}
            if (!scan_msg(base, hashed, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg w) {
                    if (!ok || (!Reads && g != 2 && g != 3)) return;
                    Seg key; key.off = key.len = 0;                   // KVReadHash{key_hash = 1, version = 2} (Reads)
                    if (!scan_msg(base, w, g == 2 ? BD_F(1) | BD_F(3) : BD_F(1) | BD_F(2), g == 2 ? BD_F(2) | BD_F(4) : 0, [&](uint32_t h, Seg k) { if (h == 1) key = k; })) { ok = false; return; }
                    if constexpr (Reads) { if (!on_write(name, cname, key, 10 + g, w)) ok = false; }
                    else on_write(name, cname, key, g == 3);
                })) ok = false;
        });
    });
    return top && ok;
}

// Appends the write records of transaction t (gone: only its metadata writes, for a transaction that never reaches VSCC) and enters its
// metadata records into the metadata-write set.
BD_HD void kl_emit(const uint8_t* base, Seg results, uint32_t t, TxDev& tx, KlArrays& kl, bool gone)
{
    uint32_t n = 0;
    if (!kl_scan_rwset(base, results, [&](Seg, Seg, Seg, bool md) { if (md || !gone) n++; })) {
        if (!gone) tx.kl_bad = 1;                                     // (a gone transaction's broken read/write set registers nothing, vpmanagerimpl.go:261-285)
        return;
    }
    if (n == 0) return;
    const uint32_t b = kl_atomic_add(kl.counter, n);
    if (b + n > kl.W_cap || b + n < b) return;                        // overflow: the decide stage sees counter[0] > W_cap
    tx.first_w = b; tx.n_w = n;
    uint32_t q = b;
    kl_scan_rwset(base, results, [&](Seg ns, Seg coll, Seg key, bool md) {
        if (!md && gone) return;
        WriteRec& w = kl.w[q];
        w.ns = ns; w.coll = coll; w.key = key; w.tx = t; w.slot = 0xffffffffu; w.md = md ? 1 : 0; w.gone = gone ? 1 : 0; w.alias = 0; w.ns_idx = 0;
        for (uint32_t k = 0; !gone && k < tx.n_ns; k++) if (seg_equal(base, tx.wr_ns[k], ns)) { w.ns_idx = (uint8_t)k; break; }
        if (md) {
            const uint64_t h = kl_rec_hash(base, w);
            bool placed = false;
            for (uint32_t probe = 0, pos = (uint32_t)h & (kl.md_size - 1); probe < kl.md_size; probe++, pos = (pos + 1) & (kl.md_size - 1)) {
#if defined(__CUDA_ARCH__)
                const uint64_t old = atomicCAS(reinterpret_cast<unsigned long long*>(kl.md_hash + pos), 0ull, (unsigned long long)h);
#else
                const uint64_t old = kl.md_hash[pos]; if (old == 0) kl.md_hash[pos] = h;
#endif
                if (old != 0 && old != h) continue;
                const unsigned long long me = ((unsigned long long)t << 32) | q;
#if defined(__CUDA_ARCH__)
                atomicMin(kl.md_min + pos, me);
#else
                if (me < kl.md_min[pos]) kl.md_min[pos] = me;
#endif
                w.slot = pos;
                placed = true; break;
            }
            if (!placed) kl.counter[1] = 1;
        }
        q++;
    });
}

// extractDependenciesForTx (validator_keylevel.go:183-221) for a transaction the walk abandoned before dispatch_plan: the levels down to
// ChaincodeAction.results, parsed as proto.Unmarshal parses them, whatever the header says.  A level that does not parse registers no
// dependency; no action, or an action payload without a ChaincodeEndorsedAction, is where the reference dereferences past the end
// (tx.Actions[0], cap.Action.ProposalResponsePayload) -- no dependency of that block can be trusted.
BD_HD void kl_lenient(const uint8_t* base, Seg env, uint32_t t, TxDev& tx, KlArrays& kl)
{
    auto none = [](uint32_t, Seg) {};
    Seg payload, data, hdr, a0, capb, act, prp, ext, results;
    payload.off = payload.len = data.off = data.len = hdr.off = hdr.len = a0.off = a0.len = capb.off = capb.len = 0;
    act.off = act.len = prp.off = prp.len = ext.off = ext.len = results.off = results.len = 0;
    bool has_hdr = false, has_act = false, ok = true; uint32_t n_act = 0;
    if (!scan_msg(base, env, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 1) payload = b; })) return;                 // Envelope
    if (!scan_msg(base, payload, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 1) { hdr = b; has_hdr = true; } else data = b; })) return;
    if (has_hdr && !scan_msg(base, hdr, BD_F(1) | BD_F(2), 0, none)) return;                                                      // Header
    if (!scan_msg(base, data, BD_F(1), 0, [&](uint32_t, Seg b) {                                                                     // Transaction
            if (!scan_msg(base, b, BD_F(1) | BD_F(2), 0, none)) ok = false;                                                       // TransactionAction
            if (n_act++ == 0) a0 = b; }) || !ok) return;
    if (n_act == 0) { kl.counter[1] = 1; return; }
    scan_msg(base, a0, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 2) capb = b; });
    if (!scan_msg(base, capb, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 2) { act = b; has_act = true; } })) return;   // ChaincodeActionPayload
    if (!has_act) { kl.counter[1] = 1; return; }
    if (!scan_msg(base, act, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) {                                                          // ChaincodeEndorsedAction
            if (f == 1) prp = b; else if (!scan_msg(base, b, BD_F(1) | BD_F(2), 0, none)) ok = false; }) || !ok) return;           // Endorsement
    if (!scan_msg(base, prp, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 2) ext = b; })) return;                        // ProposalResponsePayload
    if (!scan_msg(base, ext, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t f, Seg b) {                                    // ChaincodeAction
            if (f == 1) results = b;
            else if (f == 3) ok = ok && scan_msg(base, b, BD_F(2) | BD_F(3), BD_F(1), none);                                        // Response
            else if (f == 4) ok = ok && scan_msg(base, b, BD_F(1) | BD_F(2) | BD_F(3), 0, none); }) || !ok) return;                  // ChaincodeID
    kl_emit(base, results, t, tx, kl, true);
}

// alloc_end(n) must return the first index of n fresh endorsement-job slots (atomicAdd on the device, a counter on the host)
template <typename Alloc>
BD_HD void walk_tx_core(const uint8_t* base, Seg env, uint32_t t, const uint8_t* channel, uint32_t channel_len, TxDev& tx, RawJob* raw,
                        JobArrays& ja, Alloc alloc_end)
{
    tx.early = TXC_NOT_VALIDATED; tx.htype = 0; tx.endorser_parse_ok = 0; tx.channel_ok = 0; tx.endorsements_parse_ok = 1; tx.overflow = 0;
    tx.disp = TXC_VALID; tx.n_ns = 0; tx.n_coll = 0; tx.pub_ns = 0; tx.creator_identity = -1; tx.creator_has_job = 0; tx.first_end_job = 0; tx.n_end_jobs = 0;
    tx.txid_ascii.off = tx.txid_ascii.len = 0; tx.phash_claimed.off = tx.phash_claimed.len = 0;
    tx.results.off = tx.results.len = 0; tx.first_w = tx.n_w = 0; tx.kl_bad = 0; tx.v13_sys = BD_SYS_APP; tx.r_ver.off = tx.r_ver.len = 0;
    {
        ShaJobD z; for (int k = 0; k < 3; k++) { z.off[k] = 0; z.len[k] = 0; }
        ja.sha[t] = z; ja.sha[ja.J_cap + 2 * t] = z; ja.sha[ja.J_cap + 2 * t + 1] = z;
        raw[t].tx = 0xffffffffu; raw[t].k = -1;
    }
    Sel e = make_sel(1, 2);                                           // Envelope{payload=1, signature=2}
    if (!parse_sel(base, env, e)) { tx.early = TXC_INVALID_OTHER_REASON; return; }
    const Seg payload = e.s[0], signature = e.s[1];
    Sel p = make_sel(1, 2);                                           // Payload{header=1, data=2}
    if (!parse_sel(base, payload, p)) { tx.early = TXC_BAD_PAYLOAD; return; }
    if (!p.present[0]) { tx.early = TXC_BAD_COMMON_HEADER; return; }
    const Seg data = p.s[1]; const bool has_data = p.present[1];
    Sel h = make_sel(1, 2);                                           // Header{channel_header=1, signature_header=2}
    if (!parse_sel(base, p.s[0], h)) { tx.early = TXC_BAD_COMMON_HEADER; return; }
    const Seg chdr_b = h.s[0], shdr_b = h.s[1]; const bool has_chdr = h.present[0];
    Sel ch = make_sel(4, 5, 7, 1, 6);                                 // ChannelHeader{type=1, channel_id=4, tx_id=5, epoch=6, extension=7}
    if (!parse_sel(base, chdr_b, ch)) { tx.early = TXC_BAD_COMMON_HEADER; return; }
    Sel sh = make_sel(1, 2);                                          // SignatureHeader{creator=1, nonce=2}
    if (!parse_sel(base, shdr_b, sh)) { tx.early = TXC_BAD_COMMON_HEADER; return; }
    const Seg creator = sh.s[0], nonce = sh.s[1];
    const uint32_t ht = (uint32_t)ch.uv[0];
    if (!(ht == 1 || ht == 2 || ht == 3) || ch.uv[1] != 0 || nonce.len == 0 || creator.len == 0) { tx.early = TXC_BAD_COMMON_HEADER; return; }
    tx.htype = (uint8_t)ht;
    if (signature.len > 0 && payload.len > 0) {                       // creator job: slot t (identity resolved per job)
        raw[t].ident = creator; raw[t].sig = signature; raw[t].tx = t; raw[t].k = -1;
        ShaJobD& sj = ja.sha[t]; sj.off[0] = payload.off; sj.len[0] = payload.len;
        tx.creator_has_job = 1;
    }
    if (ht != 3) return;
    tx.txid_ascii = ch.s[1];
    { ShaJobD& a = ja.sha[ja.J_cap + 2 * t]; a.off[0] = nonce.off; a.len[0] = nonce.len; a.off[1] = creator.off; a.len[1] = creator.len; }
    tx.channel_ok = (ch.s[0].len == channel_len && bytes_equal(base + ch.s[0].off, channel, channel_len)) ? 1 : 0;
    if (!has_data) return;
    Seg action0; action0.off = action0.len = 0; uint32_t n_actions = 0;   // Transaction{repeated actions=1}: exactly one
    {
        Reader r; r.base = base; r.pos = data.off; r.end = data.off + data.len; r.ok = true;
        uint32_t f, wt; uint64_t v; Seg b;
        while (r.next(f, wt, v, b)) { if (f == 1) { if (wt != 2) { r.ok = false; break; } action0 = b; n_actions++; } }
        if (!r.ok || n_actions != 1) return;
    }
    Sel ta = make_sel(1, 2);                                          // TransactionAction{header=1, payload=2}
    if (!parse_sel(base, action0, ta)) return;
    Sel ah = make_sel(1, 2);
    if (!parse_sel(base, ta.s[0], ah) || ah.s[1].len == 0 || ah.s[0].len == 0) return;
    Sel cap = make_sel(1, 2);                                         // ChaincodeActionPayload{chaincode_proposal_payload=1, action=2}
    if (!parse_sel(base, ta.s[1], cap) || !cap.present[1]) return;
    Seg prp; prp.off = prp.len = 0; uint32_t n_end = 0; bool has_prp = false;   // ChaincodeEndorsedAction{prp=1, repeated endorsements=2}
    {
        Reader r; r.base = base; r.pos = cap.s[1].off; r.end = cap.s[1].off + cap.s[1].len; r.ok = true;
        uint32_t f, wt; uint64_t v; Seg b;
        while (r.next(f, wt, v, b)) {
            if (f == 1) { if (wt != 2) { r.ok = false; break; } prp = b; has_prp = true; }
            else if (f == 2) { if (wt != 2) { r.ok = false; break; } n_end++; }
        }
        if (!r.ok) return;
    }
    Sel pr = make_sel(1, 2);                                          // ProposalResponsePayload{proposal_hash=1, extension=2}
    if (!parse_sel(base, prp, pr)) return;
    if (!has_chdr || !ta.present[0] || !cap.present[0]) return;       // GetProposalHash2 "nil arguments"
    { ShaJobD& b = ja.sha[ja.J_cap + 2 * t + 1];
      b.off[0] = chdr_b.off; b.len[0] = chdr_b.len; b.off[1] = ta.s[0].off; b.len[1] = ta.s[0].len; b.off[2] = cap.s[0].off; b.len[2] = cap.s[0].len; }
    tx.phash_claimed = pr.s[0];
    tx.endorser_parse_ok = 1;
    dispatch_plan(base, ch.s[2], has_prp, pr.present[1], pr.s[1], tx, ja.mode);
    // key policy table installed: the writes the key-level checks walk (a transaction the dispatcher stops is walk_tx's)
    if (ja.kl.w && tx.disp == TXC_VALID) kl_emit(base, tx.results, t, tx, ja.kl, false);
    // endorsements: one pass to count those that carry a signature, one to emit their jobs (contiguous, in endorsement order)
    uint32_t n_jobs = 0;
    {
        Reader r; r.base = base; r.pos = cap.s[1].off; r.end = cap.s[1].off + cap.s[1].len; r.ok = true;
        uint32_t f, wt; uint64_t v; Seg b;
        while (r.next(f, wt, v, b)) {
            if (f != 2) continue;
            Sel en = make_sel(1, 2);                                  // Endorsement{endorser=1, signature=2}
            if (!parse_sel(base, b, en)) { tx.endorsements_parse_ok = 0; break; }
            // an endorsement without signature bytes can never verify: whatever its identity, it contributes nothing
            if (en.s[1].len > 0) n_jobs++;
        }
    }
    if (!tx.endorsements_parse_ok || n_jobs == 0) return;
    uint32_t j = alloc_end(n_jobs);
    if (j + n_jobs > ja.J_cap || j + n_jobs < j) {                    // job arrays full: this transaction goes to the CPU validator
        tx.overflow = 1;
        // The later stages run over every slot up to J_cap once the counter passes it: the slots handed out here that still
        // lie inside the arrays get dead records, not whatever the previous block (or cudaMalloc) left there.
        ShaJobD z; for (int k = 0; k < 3; k++) { z.off[k] = 0; z.len[k] = 0; }
        for (uint32_t q = j; q < ja.J_cap && q - j < n_jobs; q++) {
            raw[q].ident.off = raw[q].ident.len = raw[q].sig.off = raw[q].sig.len = 0; raw[q].tx = 0xffffffffu; raw[q].k = -1;
            ja.sha[q] = z;
        }
        return;
    }
    tx.first_end_job = j; tx.n_end_jobs = n_jobs;
    {
        Reader r; r.base = base; r.pos = cap.s[1].off; r.end = cap.s[1].off + cap.s[1].len; r.ok = true;
        uint32_t f, wt; uint64_t v; Seg b; int32_t k = 0;
        while (r.next(f, wt, v, b)) {
            if (f != 2) continue;
            Sel en = make_sel(1, 2);
            parse_sel(base, b, en);
            if (en.s[1].len == 0) continue;
            raw[j].ident = en.s[0]; raw[j].sig = en.s[1]; raw[j].tx = t; raw[j].k = k++;
            ShaJobD& sj = ja.sha[j];
            sj.off[0] = prp.off; sj.len[0] = prp.len; sj.off[1] = en.s[0].off; sj.len[1] = en.s[0].len; sj.off[2] = 0; sj.len[2] = 0;
            j++;
        }
    }
}

// The walk of one transaction.  With a key policy table, a transaction that does not reach the VSCC stage on structure alone (the walk
// or the dispatcher stops it) still registers the dependencies of its metadata writes: it never signals a result, so a later writer of
// the same key would wait for it forever (vpmanagerimpl.go:196-230).
template <typename Alloc>
BD_HD void walk_tx(const uint8_t* base, Seg env, uint32_t t, const uint8_t* channel, uint32_t channel_len, TxDev& tx, RawJob* raw,
                   JobArrays& ja, Alloc alloc_end)
{
    walk_tx_core(base, env, t, channel, channel_len, tx, raw, ja, alloc_end);
    if (ja.kl.w && !(tx.endorser_parse_ok && tx.disp == TXC_VALID)) kl_lenient(base, env, t, tx, ja.kl);
}

// One signature job: identity lookup in the MSP table, DER / low-S gate, operands for the verify kernel, and (creator jobs) the
// identity index written back into the transaction record.
BD_HD void resolve_job(const uint8_t* base, uint32_t j, const RawJob* raw, const MspDev& msp, JobArrays& ja, TxDev* txs)
{
    const RawJob rj = raw[j];
    int32_t identity = -1;
    bool ok = false;
    uint8_t rr[32], ss[32];
    if (rj.tx != 0xffffffffu) {
        identity = msp_find(msp, base + rj.ident.off, rj.ident.len);
        if (rj.k < 0) txs[rj.tx].creator_identity = identity;
        if (identity >= 0) ok = gate_signature(base + rj.sig.off, rj.sig.len, rr, ss);
    }
    uint32_t* r4 = reinterpret_cast<uint32_t*>(ja.r + 32 * (size_t)j);
    uint32_t* s4 = reinterpret_cast<uint32_t*>(ja.s + 32 * (size_t)j);
    for (int k = 0; k < 8; k++) {
        r4[k] = ok ? ((uint32_t)rr[4 * k] | ((uint32_t)rr[4 * k + 1] << 8) | ((uint32_t)rr[4 * k + 2] << 16) | ((uint32_t)rr[4 * k + 3] << 24)) : 0u;
        s4[k] = ok ? ((uint32_t)ss[4 * k] | ((uint32_t)ss[4 * k + 1] << 8) | ((uint32_t)ss[4 * k + 2] << 16) | ((uint32_t)ss[4 * k + 3] << 24)) : 0u;
    }
    ja.gate_ok[j] = ok ? 1 : 0;
    ja.identity[j] = identity;
    const int32_t slot = (identity >= 0 && ok) ? msp.key_slot[identity] : -1;
    ja.key_slot[j] = slot;
    if (identity >= 0 && ok && slot == -1 && ja.qx) {
        for (int i = 0; i < 32; i++) { ja.qx[32 * (size_t)j + i] = msp.keys_xy[64 * (size_t)identity + i]; ja.qy[32 * (size_t)j + i] = msp.keys_xy[64 * (size_t)identity + 32 + i]; }
    }
}

// One slot of the key policy table: the entry's namespace, collection and key lie back to back at kp_blob + off.  hash 0 = empty.
// root: a node of the policy array, KP_UNDECIDABLE, or KP_REMOVED.
struct KpSlot { uint64_t hash; uint32_t off, ns_len, coll_len, key_len; int32_t root; uint32_t pad; };

// ---- policy evaluator: cauthdsl.go:24-92, `used` as a bit mask over at most BD_MAX_SIGNERS signers ------------------------
// Several policies share one node array (one tree per chaincode namespace); ns_* name the root of each.
// Node types: 0 = NOutOf(n), 1 = SignedBy(principal n), 2 = ImplicitMeta with threshold n (implicitmeta.go:69-103).
// principal_bits (fabgpu_msp_principal_bits): bits_words words per identity, bit p set = identity.SatisfiesPrincipal(p) == nil.
// Null: principals are MSP ids matched as ROLE MEMBER (msp_code equality of a valid identity).
struct PolicyDev {
    const int32_t* nodes; int32_t n_nodes; const int32_t* principal_code; int32_t n_principals;
    const uint8_t* ns_blob; const uint32_t* ns_off; const int32_t* ns_root; int32_t n_ns;     // n_ns = 0: one policy (root 0) for every namespace
    const uint32_t* principal_bits = nullptr; int32_t bits_words = 0;          // a PolicyDev built field by field has no bits
    // fabgpu_collection_policies: entry i maps (namespace i, collection i) to policy root coll_root[i]; an open-addressing table of
    // coll_size slots (a power of two) keyed by coll_key_hash finds it.  coll_size = 0: no table, every write falls under its
    // namespace's chaincode policy.
    const uint8_t* coll_ns_blob = nullptr; const uint32_t* coll_ns_off = nullptr; const uint8_t* coll_name_blob = nullptr;
    const uint32_t* coll_name_off = nullptr; const int32_t* coll_root = nullptr; const uint64_t* coll_hash = nullptr; const int32_t* coll_idx = nullptr;
    uint32_t coll_size = 0;
    // fabgpu_key_policies: key-level validation parameters, kp_size slots (a power of two) keyed by kl_key_hash; kp_size = 0: no table
    const KpSlot* kp_slots = nullptr; const uint8_t* kp_blob = nullptr; uint32_t kp_size = 0;
    // fabgpu_channel_capability: BD_MODE_V13 selects the v1.4 validator (decide_tx); fabgpu_namespace_versions: the lscc version of
    // namespace table entry i at ver_blob + ver_off[i] .. ver_off[i + 1] (empty: none), null = no versions
    uint8_t mode = BD_MODE_V20; const uint8_t* ver_blob = nullptr; const uint32_t* ver_off = nullptr;
};

// root of the validation parameter of (ns, coll, key) (all in the block), -1 when the table holds none
BD_HD int32_t kp_find(const PolicyDev& pol, const uint8_t* base, Seg ns, Seg coll, Seg key)
{
    const uint64_t h = kl_key_hash(base + ns.off, ns.len, base + coll.off, coll.len, base + key.off, key.len);
    for (uint32_t probe = 0, pos = (uint32_t)h & (pol.kp_size - 1); probe < pol.kp_size; probe++, pos = (pos + 1) & (pol.kp_size - 1)) {
        const KpSlot s = pol.kp_slots[pos];
        if (s.hash == 0) return -1;
        if (s.hash != h || s.ns_len != ns.len || s.coll_len != coll.len || s.key_len != key.len) continue;
        const uint8_t* e = pol.kp_blob + s.off;
        if (bytes_equal(e, base + ns.off, ns.len) && bytes_equal(e + ns.len, base + coll.off, coll.len) &&
            bytes_equal(e + ns.len + coll.len, base + key.off, key.len))
            return s.root == KP_REMOVED ? -1 : s.root;
    }
    return -1;
}

// metadata-write set entry of record w's key, 0xffffffff when no transaction of the block metadata-writes a key with its hash
BD_HD uint32_t kl_md_find(const KlArrays& kl, const uint8_t* base, const WriteRec& w)
{
    const uint64_t h = kl_rec_hash(base, w);
    for (uint32_t probe = 0, pos = (uint32_t)h & (kl.md_size - 1); probe < kl.md_size; probe++, pos = (pos + 1) & (kl.md_size - 1)) {
        const uint64_t k = kl.md_hash[pos];
        if (k == 0) return 0xffffffffu;
        if (k == h) return pos;
    }
    return 0xffffffffu;
}

// Decide stage, every transaction t (before decide_tx): marks t as a metadata writer, and an entry whose metadata writers do not all
// share its first writer's key as mixed.
BD_HD void kl_mark(const uint8_t* base, uint32_t t, const TxDev& tx, KlArrays& kl)
{
    uint8_t mark = 0;
    for (uint32_t q = 0; q < tx.n_w; q++) {
        const WriteRec& w = kl.w[tx.first_w + q];
        if (!w.md || w.slot == 0xffffffffu) continue;
        mark = 2;
        if (!kl_same_key(base, kl.w[(uint32_t)kl.md_min[w.slot]], w)) {
#if defined(__CUDA_ARCH__)
            atomicOr(kl.md_sum + w.slot, KL_SUM_MIXED);
#else
            kl.md_sum[w.slot] |= KL_SUM_MIXED;
#endif
        }
    }
    kl.conflicted[t] = mark;
}

// The resolve rule, applied to the marked transactions in index order (vpmanagerimpl.go:196-230).  A transaction t that writes a key some
// earlier transaction j metadata-wrote waits for j's VSCC result for that namespace, and fails with a policy error if any is nil.  It is
// read off j's final flag (final when t's turn comes; the duplicate-tx-id pass runs after VSCC): VALID -> nil; ENDORSEMENT_POLICY_FAILURE
// with one validated namespace (the written one) -> non-nil; anything else -> undetermined: j never reached that namespace's VSCC
// (rejected before it, or the dispatcher stopped at another namespace first, dispatcher.go:190-217) and the reference would wait
// forever -- or j is one the device did not decide.  Undetermined gives NOT_VALIDATED, else any nil gives ENDORSEMENT_POLICY_FAILURE,
// else t keeps its own decision.  Each entry's md_sum folds in its writers as they are passed, so a step costs t's own records: a key
// that every transaction of the block writes and metadata-writes costs the block O(T), not O(T^2).
BD_HD void kl_resolve_step(uint32_t t, const TxDev* txs, KlArrays& kl, uint8_t* flags)
{
    const TxDev& x = txs[t];
    const uint8_t mark = kl.conflicted[t];
    uint8_t f = flags[t];
    if ((mark & 1) && (f == TXC_VALID || f == TXC_ENDORSEMENT_POLICY_FAILURE)) {
        uint32_t s = 0;
        for (uint32_t q = 0; q < x.n_w; q++) {
            const WriteRec& w = kl.w[x.first_w + q];
            if (w.slot == 0xffffffffu) continue;
            const uint32_t u = kl.md_sum[w.slot];
            if (!(u & KL_SUM_ANY)) continue;                          // no earlier writer of this hash
            s |= (w.alias || (u & KL_SUM_MIXED)) ? KL_SUM_UNDET : (u & (KL_SUM_NIL | KL_SUM_UNDET));
        }
        f = (s & KL_SUM_UNDET) ? TXC_NOT_VALIDATED : (s & KL_SUM_NIL) ? TXC_ENDORSEMENT_POLICY_FAILURE : f;
        flags[t] = f;
    }
    if (mark & 2) {
        const bool gone = x.n_w && kl.w[x.first_w].gone;
        // (a v1.3-mode qscc / cscc invocation validates only its own namespace, whatever it metadata-writes: undetermined)
        const bool decided = !gone && x.v13_sys == BD_SYS_APP;
        const uint32_t st = KL_SUM_ANY | (f == TXC_VALID && decided ? KL_SUM_NIL
                                          : f == TXC_ENDORSEMENT_POLICY_FAILURE && x.n_ns == 1 && decided ? 0u : KL_SUM_UNDET);
        for (uint32_t q = 0; q < x.n_w; q++) {
            const WriteRec& w = kl.w[x.first_w + q];
            if (w.md && w.slot != 0xffffffffu) kl.md_sum[w.slot] |= st;
        }
    }
}

BD_HD uint64_t coll_key_hash(const uint8_t* ns, uint32_t ns_len, const uint8_t* coll, uint32_t coll_len)
{
    uint64_t h = 1469598103934665603ull ^ ns_len;
    for (uint32_t i = 0; i < ns_len; i++) h = (h ^ ns[i]) * 1099511628211ull;
    h = (h ^ coll_len) * 1099511628211ull;
    for (uint32_t i = 0; i < coll_len; i++) h = (h ^ coll[i]) * 1099511628211ull;
    return h ? h : 1;
}

// Host side of fabgpu_collection_policies: fills the table (size a power of two above n; hash all zero, idx any) with entries
// [0, n).  false when two entries name the same (namespace, collection).
inline bool coll_table_fill(const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off, int32_t n,
                            uint32_t size, uint64_t* hash, int32_t* idx)
{
    for (int32_t i = 0; i < n; i++) {
        const uint32_t nl = ns_off[i + 1] - ns_off[i], cl = coll_off[i + 1] - coll_off[i];
        const uint64_t h = coll_key_hash(ns_blob + ns_off[i], nl, coll_blob + coll_off[i], cl);
        uint32_t pos = (uint32_t)h & (size - 1);
        for (; hash[pos] != 0; pos = (pos + 1) & (size - 1)) {
            const int32_t k = idx[pos];
            if (hash[pos] == h && ns_off[k + 1] - ns_off[k] == nl && coll_off[k + 1] - coll_off[k] == cl &&
                memcmp(ns_blob + ns_off[k], ns_blob + ns_off[i], nl) == 0 && memcmp(coll_blob + coll_off[k], coll_blob + coll_off[i], cl) == 0)
                return false;
        }
        hash[pos] = h; idx[pos] = i;
    }
    return true;
}

// policy root of collection `coll` of namespace `ns` (both in the block), -1 when the table has no entry for it
BD_HD int32_t coll_policy_root(const PolicyDev& pol, const uint8_t* base, Seg ns, Seg coll)
{
    const uint64_t h = coll_key_hash(base + ns.off, ns.len, base + coll.off, coll.len);
    for (uint32_t probe = 0, pos = (uint32_t)h & (pol.coll_size - 1); probe < pol.coll_size; probe++, pos = (pos + 1) & (pol.coll_size - 1)) {
        const uint64_t k = pol.coll_hash[pos];
        if (k == 0) return -1;
        if (k != h) continue;
        const int32_t i = pol.coll_idx[pos];
        const uint32_t no = pol.coll_ns_off[i], co = pol.coll_name_off[i];
        if (pol.coll_ns_off[i + 1] - no == ns.len && pol.coll_name_off[i + 1] - co == coll.len &&
            bytes_equal(pol.coll_ns_blob + no, base + ns.off, ns.len) && bytes_equal(pol.coll_name_blob + co, base + coll.off, coll.len))
            return pol.coll_root[i];
    }
    return -1;
}

// signer[i]: with principal bits, the identity index of verified signer i; without, its MSP-id code, -1 when Validate() failed.
BD_HD bool eval_policy(const PolicyDev& pol, int idx, const int32_t* signer, int n_signers, uint64_t& used, int depth)
{
    if (idx < 0 || idx >= pol.n_nodes || depth > BD_MAX_POLICY_DEPTH) return false;
    const int32_t type = pol.nodes[4 * idx], n = pol.nodes[4 * idx + 1], first = pol.nodes[4 * idx + 2], cnt = pol.nodes[4 * idx + 3];
    if (type == 0) {
        int verified = 0;
        for (int c = first; c < first + cnt; c++) {
            uint64_t scratch = used;
            if (eval_policy(pol, c, signer, n_signers, scratch, depth + 1)) { verified++; used = scratch; }
        }
        return verified >= n;
    }
    if (type == 2) {
        // Every sub-policy is a policy of its own (its own SignatureSetToValidIdentities and cauthdsl `used`): one signer may satisfy
        // several of them, and the caller's `used` is not touched.
        int satisfied = 0;
        for (int c = first; c < first + cnt && satisfied < n; c++) {
            uint64_t fresh = 0;
            if (eval_policy(pol, c, signer, n_signers, fresh, depth + 1)) satisfied++;
        }
        return satisfied >= n;
    }
    if (type != 1 || n < 0 || n >= pol.n_principals) return false;
    if (pol.principal_bits) {
        const uint32_t word = (uint32_t)n >> 5, bit = 1u << (n & 31);
        for (int i = 0; i < n_signers; i++) {
            if (used & (1ull << i)) continue;
            if (!(pol.principal_bits[(size_t)signer[i] * pol.bits_words + word] & bit)) continue;
            used |= 1ull << i;
            return true;
        }
        return false;
    }
    const int32_t want = pol.principal_code[n];
    for (int i = 0; i < n_signers; i++) {
        if (used & (1ull << i)) continue;
        if (signer[i] < 0 || signer[i] != want) continue;
        used |= 1ull << i;
        return true;
    }
    return false;
}

// entry of namespace `ns` in the namespace table, -1 when it has none
BD_HD int32_t policy_index(const PolicyDev& pol, const uint8_t* base, Seg ns)
{
    for (int32_t i = 0; i < pol.n_ns; i++) {
        const uint32_t o = pol.ns_off[i], l = pol.ns_off[i + 1] - o;
        if (l != ns.len) continue;
        bool eq = true;
        for (uint32_t k = 0; k < l && eq; k++) eq = pol.ns_blob[o + k] == base[ns.off + k];
        if (eq) return i;
    }
    return -1;
}

// root node of namespace `ns`'s policy, -1 when the table has no chaincode definition for it
BD_HD int32_t policy_root(const PolicyDev& pol, const uint8_t* base, Seg ns)
{
    if (pol.n_ns == 0) return pol.n_nodes > 0 ? 0 : -1;
    const int32_t i = policy_index(pol, base, ns);
    return i < 0 ? -1 : pol.ns_root[i];
}

// SignatureSetToValidIdentities (policy.go:365-402): in order; de-duplicated by Mspid + Id against the identities that already
// VERIFIED; a failed signature drops that entry only.  One set per transaction, shared by every namespace's evaluation.
// With principal bits a signer is its identity index: the caller's SatisfiesPrincipal answers already include Validate() where
// the reference checks it (an admin-listed identity satisfies ADMIN without it, mspimpl.go:506-513).  Without, it is its MSP-id
// code, -1 when Validate() failed (ROLE MEMBER, mspimpl.go:501-505).  false: not decided here (an endorser the table does not hold,
// or more signers than BD_MAX_SIGNERS).
template <typename SigOk>
BD_HD bool signer_set(const TxDev& tx, const MspDev& msp, const PolicyDev& pol, SigOk sig_ok, const int32_t* job_identity, int32_t* signer,
                      int& n_signers)
{
    n_signers = 0;
    for (uint32_t i = 0; i < tx.n_end_jobs; i++) {
        const uint32_t j = tx.first_end_job + i;
        const int32_t idn = job_identity[j];
        if (idn < 0) return false;
        const int32_t grp = msp.group ? msp.group[idn] : idn;
        bool dup = false;
        for (uint32_t i2 = 0; i2 < i && !dup; i2++) {
            const uint32_t j2 = tx.first_end_job + i2;
            const int32_t id2 = job_identity[j2];
            dup = (msp.group ? msp.group[id2] : id2) == grp && sig_ok(j2);
        }
        if (dup) continue;
        if (!sig_ok(j)) continue;
        if (n_signers >= BD_MAX_SIGNERS) return false;
        signer[n_signers++] = pol.principal_bits ? idn : msp.valid[idn] ? msp.msp_code[idn] : -1;
    }
    return true;
}

// An earlier metadata write of a key t writes: marks t for the resolve stage (kl_resolve_step)
BD_HD void kl_mark_deps(const uint8_t* base, const TxDev& tx, uint32_t t, KlArrays* kl)
{
    bool dep = false;
    for (uint32_t q = 0; q < tx.n_w; q++) {
        WriteRec& w = kl->w[tx.first_w + q];
        if (!w.md) w.slot = kl_md_find(*kl, base, w);
        if (w.slot == 0xffffffffu) continue;
        const unsigned long long m = kl->md_min[w.slot];
        if ((uint32_t)(m >> 32) >= t) continue;                       // every metadata writer of this hash comes later
        dep = true;
        if (!kl_same_key(base, kl->w[(uint32_t)m], w)) w.alias = 1;
    }
    if (dep) kl->conflicted[t] |= 1;
}

BD_HD uint64_t txid_hash(const uint8_t* base, const TxDev& tx)
{
    uint64_t hsh = 1469598103934665603ull;
    for (uint32_t k = 0; k < tx.txid_ascii.len; k++) hsh = (hsh ^ base[tx.txid_ascii.off + k]) * 1099511628211ull;
    return hsh;
}

// The v1.4 validator's VSCC stage (v14/vscc_validator.go:117-229,230-270 with builtin/v13): the validated namespaces in order -- the
// invoked chaincode, then the others in read/write-set order -- and the first that fails decides.  Per namespace: its table entry
// (none: 254), for the invoked application chaincode the lscc version (:195-208; none installed: 254, another: EXPIRED_CHAINCODE),
// then its own writes only (baseEvaluator.Evaluate, statebased/v13.go): the key's validation parameter if it has one, otherwise the
// chaincode policy -- no collection policies.  A namespace without writes is checked against its chaincode policy.
template <typename SigOk>
BD_HD uint8_t decide_v13(const uint8_t* base, const TxDev& tx, uint32_t t, const MspDev& msp, const PolicyDev& pol, SigOk sig_ok,
                         const int32_t* job_identity, uint64_t* txid_hash_out, KlArrays* kl)
{
    const bool keylevel = kl && pol.kp_size;
    if (keylevel) {
        if (kl->counter[0] > kl->W_cap || kl->counter[1] || tx.kl_bad) return TXC_NOT_VALIDATED;
        for (uint32_t q = 0; q < tx.n_w; q++)                         // a qscc / cscc invocation writing elsewhere: not decided here
            if (tx.v13_sys != BD_SYS_APP && !seg_equal(base, kl->w[tx.first_w + q].ns, tx.wr_ns[0])) return TXC_NOT_VALIDATED;
    }
    int32_t signer[BD_MAX_SIGNERS]; int n_signers = -1;              // built at the first policy evaluation
    for (int i = 0; i < tx.n_ns; i++) {
        const int32_t cc_root = policy_root(pol, base, tx.wr_ns[i]);
        if (cc_root < 0) return TXC_NOT_VALIDATED;
        if (i == 0 && tx.v13_sys == BD_SYS_APP) {
            const int32_t k = pol.ver_off ? policy_index(pol, base, tx.wr_ns[0]) : -1;
            const uint32_t vo = k < 0 ? 0 : pol.ver_off[k], vl = k < 0 ? 0 : pol.ver_off[k + 1] - vo;
            if (vl == 0) return TXC_NOT_VALIDATED;                    // no lscc version on the device
            if (vl != tx.r_ver.len || !bytes_equal(pol.ver_blob + vo, base + tx.r_ver.off, vl)) return TXC_EXPIRED_CHAINCODE;
        }
        int32_t need[BD_MAX_NEED]; int n_need = 0; bool too_many = false;
        auto add = [&](int32_t r) {
            for (int k = 0; k < n_need; k++) if (need[k] == r) return;
            if (n_need == BD_MAX_NEED) too_many = true; else need[n_need++] = r;
        };
        bool wrote = false;
        for (uint32_t q = 0; keylevel && q < tx.n_w; q++) {
            const WriteRec& w = kl->w[tx.first_w + q];
            if (w.ns_idx != i) continue;
            const int32_t cr = w.coll.len && pol.coll_size ? coll_policy_root(pol, base, w.ns, w.coll) : -1;
            if (w.coll.len && pol.coll_size && cr < 0) return TXC_NOT_VALIDATED;   // as in v2.0 mode: the collection may be undefined
            const int32_t r = kp_find(pol, base, w.ns, w.coll, w.key);
            if (r == KP_UNDECIDABLE) return TXC_NOT_VALIDATED;
            add(r < 0 ? cc_root : r);
            wrote = true;
        }
        if (!wrote) add(cc_root);
        if (too_many) return TXC_NOT_VALIDATED;
        if (n_signers < 0 && !signer_set(tx, msp, pol, sig_ok, job_identity, signer, n_signers)) return TXC_NOT_VALIDATED;
        bool pass = true;
        for (int k = 0; k < n_need && pass; k++) {
            uint64_t used = 0;
            pass = eval_policy(pol, need[k], signer, n_signers, used, 0);
        }
        if (!pass) {
            if (keylevel) kl_mark_deps(base, tx, t, kl);
            return TXC_ENDORSEMENT_POLICY_FAILURE;
        }
    }
    if (keylevel) kl_mark_deps(base, tx, t, kl);
    *txid_hash_out = txid_hash(base, tx);
    return TXC_VALID;
}

// ---- per-transaction decision ---------------------------------------------------------------------------------------------
// sig_ok(j): signature job j verified (gate and curve).  job_identity: JobArrays::identity.  digests: 32 bytes per SHA job.
// An identity the table does not hold, a namespace without a policy entry, or (with a collection table) a written collection without
// one, cannot be decided here: TXC_NOT_VALIDATED hands the
// transaction to the CPU validator (the reference deserialises and validates ANY certificate of the channel's CAs,
// msgvalidation.go:40-57, and reads chaincode definitions from the ledger, dispatcher.go:224-277).
// kl: the block's write records and metadata-write set, used while a key policy table is installed (pol.kp_size != 0); decide_tx then
// sets bit 0 of kl->conflicted[t] when an earlier transaction metadata-wrote a key t writes, for the resolve stage (kl_resolve_step).
// txids: the committed tx-id set (fabgpu_committed_txids), null = none installed.
template <typename SigOk>
BD_HD uint8_t decide_tx(const uint8_t* base, const TxDev& tx, uint32_t t, const MspDev& msp, const PolicyDev& pol, SigOk sig_ok,
                        const int32_t* job_identity, const uint8_t* digests, uint32_t J_cap, uint64_t* txid_hash_out, KlArrays* kl = nullptr,
                        const TxidSetDev* txids = nullptr)
{
    const char hex[] = "0123456789abcdef";
    if (tx.early != TXC_NOT_VALIDATED) return tx.early;
    if (!tx.creator_has_job) return TXC_BAD_CREATOR_SIGNATURE;        // "nil arguments"
    if (tx.creator_identity < 0) return TXC_NOT_VALIDATED;            // not in the device's MSP table
    if (!msp.valid[tx.creator_identity] || !sig_ok(t)) return TXC_BAD_CREATOR_SIGNATURE;
    if (tx.htype == 1) return TXC_NOT_VALIDATED;                      // config transaction: CPU validator
    if (tx.htype != 3) return TXC_UNSUPPORTED_TX_PAYLOAD;
    {
        const uint8_t* dg = digests + 32 * (size_t)(J_cap + 2 * t);
        bool same = tx.txid_ascii.len == 64;
        for (int k = 0; same && k < 32; k++)
            same = base[tx.txid_ascii.off + 2 * k] == (uint8_t)hex[dg[k] >> 4] && base[tx.txid_ascii.off + 2 * k + 1] == (uint8_t)hex[dg[k] & 15];
        if (!same) return TXC_BAD_PROPOSAL_TXID;
    }
    if (!tx.endorser_parse_ok) return TXC_INVALID_ENDORSER_TRANSACTION;
    if (tx.phash_claimed.len != 32 || !bytes_equal(base + tx.phash_claimed.off, digests + 32 * (size_t)(J_cap + 2 * t + 1), 32))
        return TXC_INVALID_ENDORSER_TRANSACTION;
    if (!tx.channel_ok) return TXC_TARGET_CHAIN_NOT_FOUND;
    if (txids) {                                                      // checkTxIdDupsLedger, both validators: the id is the CheckTxID digest
        const uint32_t st = txid_lookup(*txids, digests + 32 * (size_t)(J_cap + 2 * t));
        if (st == TXID_COMMITTED) return TXC_DUPLICATE_TXID;
        if (st == TXID_UNANSWERABLE) return TXC_NOT_VALIDATED;        // GetTransactionByID fails: a terminal error of the reference's block
    }
    if (tx.disp != TXC_VALID) return tx.disp;                         // the plugin dispatcher's own checks
    if (!tx.endorsements_parse_ok) return TXC_INVALID_OTHER_REASON;
    if (tx.overflow) return TXC_NOT_VALIDATED;                        // job arrays were full: CPU validator
    if (pol.mode == BD_MODE_V13) return decide_v13(base, tx, t, msp, pol, sig_ok, job_identity, txid_hash_out, kl);
    // The policies to satisfy, each root once (evaluation has no state across policies, so the reference's nsEPChecked memo,
    // v20.go:105-147, changes no outcome).  Without a collection table: every validated namespace's chaincode policy.  With one, per
    // namespace as baseEvaluator.Evaluate (validator_keylevel.go:86-142) walks its writes: the collection's policy for each named
    // collection written, the chaincode policy for public writes and collections without a name, and the chaincode policy when
    // nothing else was checked (CheckCCEPIfNoEPChecked, v20.go:149-163: the invoked chaincode that only reads).
    int32_t roots[BD_MAX_NS], need[BD_MAX_NEED]; int n_need = 0; bool too_many = false;
    auto add = [&](int32_t r) {
        for (int k = 0; k < n_need; k++) if (need[k] == r) return;
        if (n_need == BD_MAX_NEED) too_many = true; else need[n_need++] = r;
    };
    for (int i = 0; i < tx.n_ns; i++) {
        roots[i] = policy_root(pol, base, tx.wr_ns[i]);
        if (roots[i] < 0) return TXC_NOT_VALIDATED;                   // no chaincode definition on the device
    }
    const bool keylevel = kl && pol.kp_size;
    if (keylevel) {
        // checkSBAndCCEP per write (validator_keylevel.go:37-84): the key's validation parameter if it has one (and then not the
        // chaincode's or collection's policy for that write), else CheckCCEPIfNotChecked; CheckCCEPIfNoEPChecked for a namespace none
        // of whose writes checked anything -- one without writes, since every write checks something.
        if (kl->counter[0] > kl->W_cap || kl->counter[1] || tx.kl_bad) return TXC_NOT_VALIDATED;   // records lost, or unreadable
        uint32_t has_w = 0;
        for (uint32_t q = 0; q < tx.n_w; q++) {
            const WriteRec& w = kl->w[tx.first_w + q];
            // With a collection table, a collection it does not hold may be one the chaincode does not define, where the reference skips
            // the key's parameter (CollConfigNotDefinedError, validator_keylevel.go:53-54) and then fails: not decided here, VP or not.
            const int32_t cr = w.coll.len && pol.coll_size ? coll_policy_root(pol, base, w.ns, w.coll) : -1;
            if (w.coll.len && pol.coll_size && cr < 0) return TXC_NOT_VALIDATED;
            int32_t r = kp_find(pol, base, w.ns, w.coll, w.key);
            if (r == KP_UNDECIDABLE) return TXC_NOT_VALIDATED;
            if (r < 0) r = w.coll.len && pol.coll_size ? cr : roots[w.ns_idx];
            add(r);
            has_w |= 1u << w.ns_idx;
        }
        for (int i = 0; i < tx.n_ns; i++) if (!((has_w >> i) & 1u)) add(roots[i]);
        if (too_many) return TXC_NOT_VALIDATED;
    } else if (pol.coll_size == 0) {
        for (int i = 0; i < tx.n_ns; i++) add(roots[i]);
    } else {
        if (tx.n_coll > BD_MAX_COLL) return TXC_NOT_VALIDATED;          // more collections than the walk records
        uint32_t has_coll = 0;
        for (int c = 0; c < tx.n_coll; c++) {
            const int32_t r = coll_policy_root(pol, base, tx.wr_ns[tx.coll_ns[c]], tx.coll[c]);
            if (r < 0) return TXC_NOT_VALIDATED;                        // CollectionValidationInfo would read the ledger
            add(r);
            has_coll |= 1u << tx.coll_ns[c];
        }
        for (int i = 0; i < tx.n_ns; i++)
            if (((tx.pub_ns | ~has_coll) >> i) & 1u) add(roots[i]);
    }
    int32_t signer[BD_MAX_SIGNERS]; int n_signers = 0;
    if (!signer_set(tx, msp, pol, sig_ok, job_identity, signer, n_signers)) return TXC_NOT_VALIDATED;
    bool pass = true;
    for (int k = 0; k < n_need && pass; k++) {
        uint64_t used = 0;
        pass = eval_policy(pol, need[k], signer, n_signers, used, 0);
    }
    if (keylevel) kl_mark_deps(base, tx, t, kl);                      // an earlier metadata write of a key t writes: resolved later
    if (!pass) return TXC_ENDORSEMENT_POLICY_FAILURE;
    *txid_hash_out = txid_hash(base, tx);
    return TXC_VALID;
}

// v1.3 mode, after decide_tx: a transaction invoking lscc that the device flags 254 -- at its lscc check, or earlier (a creator outside the
// table, more namespaces than the walk records, ...) -- may be an upgrade the reference accepts, which then invalidates the block's later
// invocations of that chaincode (v14/validator.go:210-220,487-530).  Sets *lscc_seen: every VALID flag of the block becomes 254.
BD_HD void lscc_mark(const TxDev& tx, uint8_t flag, uint32_t* lscc_seen)
{
    if (tx.v13_sys == BD_SYS_LSCC && flag == TXC_NOT_VALIDATED) *lscc_seen = 1;
}

} }  // namespace fabgpu::bdev
