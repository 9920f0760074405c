// TEST HELPER (not product code): fabgpu_committed_txids_add_block in the tests' host build -- the id extractor and the block insert
// (txidblock.cuh) that txid_block_id_kernel / txid_block_insert_kernel run, one transaction at a time, on blockdev_txid.inc's host set.
// The device hashes nonce || creator with sha256.cuh; here a plain SHA-256 does.  Built as a library of its own.
#include "blockdev_txid_host.cpp"
#include "../../fabric-mod_b200/csrc/txidblock.cuh"

namespace {

void sha256(const uint8_t* a, size_t na, const uint8_t* b, size_t nb, uint8_t out[32])
{
    static const uint32_t K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
        0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
        0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
        0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
        0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
        0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    std::vector<uint8_t> m(a, a + na);
    m.insert(m.end(), b, b + nb);
    const uint64_t bits = 8 * (uint64_t)m.size();
    m.push_back(0x80);
    while (m.size() % 64 != 56) m.push_back(0);
    for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(bits >> (8 * i)));
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    auto rotr = [](uint32_t x, int n) { return (x >> n) | (x << (32 - n)); };
    for (size_t o = 0; o < m.size(); o += 64) {
        uint32_t w[64];
        for (int i = 0; i < 16; i++) w[i] = (uint32_t)m[o + 4 * i] << 24 | (uint32_t)m[o + 4 * i + 1] << 16 | (uint32_t)m[o + 4 * i + 2] << 8 | m[o + 4 * i + 3];
        for (int i = 16; i < 64; i++)
            w[i] = w[i - 16] + (rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3)) + w[i - 7] + (rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10));
        uint32_t v[8];
        for (int i = 0; i < 8; i++) v[i] = h[i];
        for (int i = 0; i < 64; i++) {
            const uint32_t t1 = v[7] + (rotr(v[4], 6) ^ rotr(v[4], 11) ^ rotr(v[4], 25)) + ((v[4] & v[5]) ^ (~v[4] & v[6])) + K[i] + w[i];
            const uint32_t t2 = (rotr(v[0], 2) ^ rotr(v[0], 13) ^ rotr(v[0], 22)) + ((v[0] & v[1]) ^ (v[0] & v[2]) ^ (v[1] & v[2]));
            for (int k = 7; k > 0; k--) v[k] = v[k - 1];
            v[4] += t1; v[0] = t1 + t2;
        }
        for (int i = 0; i < 8; i++) h[i] += v[i];
    }
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(h[i / 4] >> (24 - 8 * (i % 4)));
}

// txid_block_id_kernel's record of transaction t
TxidSlot id_record(const uint8_t* base, const uint32_t* env_off, uint32_t t, int* kind)
{
    Seg env; env.off = env_off[t]; env.len = env_off[t + 1] - env_off[t];
    uint32_t w[8] = {0, 0, 0, 0, 0, 0, 0, 0}; Seg nonce, creator;
    nonce.off = nonce.len = creator.off = creator.len = 0;
    *kind = txid_block_extract(base, env, w, nonce, creator);
    if (*kind == TXB_COMPUTE) {
        uint8_t d[32];
        sha256(base + nonce.off, nonce.len, base + creator.off, creator.len, d);
        txid_words(d, w);
    }
    TxidSlot r;
    for (int q = 0; q < 8; q++) r.w[q] = *kind == TXB_NONE ? 0u : w[q];
    r.state = *kind == TXB_NONE ? (uint32_t)TXID_EMPTY : (uint32_t)TXID_COMMITTED;
    return r;
}

}  // namespace

extern "C" {

// Per transaction of the envelopes (T + 1 offsets into blob): kind[t] = TXB_NONE / TXB_ID / TXB_COMPUTE, ids[32 t ..] its 32 bytes
void txb_extract(const uint8_t* blob, size_t blob_len, const uint32_t* env_off, uint32_t T, uint8_t* kind, uint8_t* ids)
{
    std::vector<uint8_t> base(blob, blob + blob_len);
    base.resize(blob_len + 64, 0);
    for (uint32_t t = 0; t < T; t++) {
        int k = 0;
        const TxidSlot r = id_record(base.data(), env_off, t, &k);
        kind[t] = (uint8_t)k;
        for (int q = 0; q < 8; q++)
            for (int b = 0; b < 4; b++) ids[32 * t + 4 * q + b] = (uint8_t)(r.w[q] >> (8 * b));
    }
}

// fabgpu_committed_txids_add_block on the host set: the library's refusals of the set's state, growth for T more ids, then each
// transaction's record and insert.  Null, or the refusal / failure text (*failed as txs_apply); *inserting = transactions that inserted.
const char* txs_add_block(void* p, const uint8_t* blob, size_t blob_len, const uint32_t* env_off, uint32_t T, unsigned long long max_bytes,
                          int* failed, unsigned* inserting)
{
    TS* s = (TS*)p;
    *failed = 0; *inserting = 0;
    if (!s->installed) return "no committed tx-id set installed: call fabgpu_committed_txids first";
    if (s->broken) return "the committed tx-id set is broken by a failed call: replace it with fabgpu_committed_txids";
    if (T == 0) return nullptr;
    const uint64_t cap = max_bytes ? max_bytes : ~0ull;
    const uint64_t want = fabgpu::txid::slots_for(s->count + T, s->table.size());
    if (want != s->table.size()) {
        if (want * sizeof(TxidSlot) > cap) {
            s->broken = true; s->table.clear(); *failed = 1;
            return "committed tx-id table exceeds FABGPU_TXID_MAX_BYTES";
        }
        std::vector<TxidSlot> nt(want);
        memset(nt.data(), 0, want * sizeof(TxidSlot));
        for (const TxidSlot& o : s->table)
            if (o.state >= TXID_COMMITTED && txid_insert(nt.data(), (uint32_t)(want - 1), s->seed, o.w, o.state) < 0) { *failed = 1; return "rehash: no free slot"; }
        s->table.swap(nt);
    }
    std::vector<uint8_t> base(blob, blob + blob_len);
    base.resize(blob_len + 64, 0);
    std::vector<TxidSlot> rec(T);
    for (uint32_t t = 0; t < T; t++) { int k; rec[t] = id_record(base.data(), env_off, t, &k); }
    uint32_t dd = 64;
    while (dd < 2 * (uint64_t)T) dd <<= 1;
    std::vector<uint32_t> idx(dd, 0);
    for (uint32_t t = 0; t < T; t++) {
        int added = 0;
        const int r = txid_block_insert(s->table.data(), (uint32_t)(s->table.size() - 1), s->seed, rec.data(), t, idx.data(), dd - 1, &added);
        if (r < 0) { *failed = 1; return "insert: no free slot"; }
        *inserting += (unsigned)r;
        s->count += (unsigned long long)added;
    }
    return nullptr;
}

}  // extern "C"
