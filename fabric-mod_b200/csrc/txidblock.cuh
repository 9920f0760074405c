// fabgpu_committed_txids_add_block: the ids the block store indexes for a submitted block, extracted and inserted on the device.
//
// The block store indexes, for every transaction of a committed block whatever its flag, the id protoutil.GetOrComputeTxIDFromEnvelope
// returns (common/ledger/blkstorage/block_serialization.go:101-107, blockindex.go:112-138; protoutil/txutils.go:485-515):
//   Envelope -> Payload -> Header (a nil header fails) -> ChannelHeader; a non-empty tx_id is the id, whatever the header type, epoch
//   or channel, and the signature header is not read; otherwise the SignatureHeader is unmarshalled and the id is
//   hex(SHA-256(nonce || creator)) (ComputeTxID), even for an empty nonce or creator.  Any unmarshal failure gives "" (nothing the set
//   can hold).
// The messages are read with the walk's parse_sel and the walk's field selections, so the id path parses exactly what the block walk
// parses.  The set keeps only canonical ids; a computed id always is one.
//
// Two kernels, both after the slot's block_decide_kernel on the set's stream: txid_block_id_kernel (one thread per transaction: the
// record of its id, hashing nonce || creator itself -- such transactions are rare, and hashing here leaves the walk and its job arrays
// as they are) and txid_block_insert_kernel (one thread per transaction: the block's first transaction with an id inserts it, through
// txid_insert's claim / publish protocol and seeded probe; later ones with the same id drop out on a block-local index, since
// txid_insert must never run twice on one id at once).
#pragma once

namespace fabgpu { namespace bdev {

enum : int { TXB_NONE = 0, TXB_ID = 1, TXB_COMPUTE = 2 };

// TXB_NONE: the envelope indexes no id the set can hold.  TXB_ID: w = the 32 bytes of its canonical tx_id.  TXB_COMPUTE: the id is
// hex(SHA-256(nonce || creator)) of the segments returned.
BD_HD int txid_block_extract(const uint8_t* base, Seg env, uint32_t w[8], Seg& nonce, Seg& creator)
{
    Sel e = make_sel(1, 2);                                           // Envelope{payload=1, signature=2}
    if (!parse_sel(base, env, e)) return TXB_NONE;
    Sel p = make_sel(1, 2);                                           // Payload{header=1, data=2}
    if (!parse_sel(base, e.s[0], p) || !p.present[0]) return TXB_NONE;
    Sel h = make_sel(1, 2);                                           // Header{channel_header=1, signature_header=2}
    if (!parse_sel(base, p.s[0], h)) return TXB_NONE;
    Sel ch = make_sel(4, 5, 7, 1, 6);                                 // ChannelHeader{type=1, channel_id=4, tx_id=5, epoch=6, extension=7}
    if (!parse_sel(base, h.s[0], ch)) return TXB_NONE;
    const Seg id = ch.s[1];
    if (id.len) {                                                     // canonical: 64 characters of [0-9a-f]
        if (id.len != 64) return TXB_NONE;
        uint8_t b[32];
        for (int i = 0; i < 32; i++) {
            int v[2];
            for (int k = 0; k < 2; k++) {
                const uint8_t c = base[id.off + 2 * i + k];
                v[k] = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1;
                if (v[k] < 0) return TXB_NONE;
            }
            b[i] = (uint8_t)(v[0] << 4 | v[1]);
        }
        txid_words(b, w);
        return TXB_ID;
    }
    Sel sh = make_sel(1, 2);                                          // SignatureHeader{creator=1, nonce=2}
    if (!parse_sel(base, h.s[1], sh)) return TXB_NONE;
    creator = sh.s[0]; nonce = sh.s[1];
    return TXB_COMPUTE;
}

// Transaction t of the block-local de-duplication: claims the first free entry of `dd` (2^k >= 2T entries, zeroed; entry = t + 1) on
// its id's probe chain unless an earlier claimant carries the same id.  Returns 1 when t inserts (its state raised, or a new id), 0 when
// it has no id or another transaction of the block inserts it, -1 when the table has no free slot; *added = 1 for a new id.
BD_HD int txid_block_insert(TxidSlot* tab, uint32_t mask, uint64_t seed, const TxidSlot* rec, uint32_t t, uint32_t* dd, uint32_t dmask, int* added)
{
    *added = 0;
    if (rec[t].state == TXID_EMPTY) return 0;
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = rec[t].w[k];
    for (uint32_t pos = (uint32_t)(txid_mix(w, seed) >> 32) & dmask;; pos = (pos + 1) & dmask) {
        uint32_t o = 0;
#if defined(__CUDA_ARCH__)
        o = atomicCAS(&dd[pos], 0u, t + 1);
#else
        __atomic_compare_exchange_n(&dd[pos], &o, t + 1, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
#endif
        if (o == 0) break;
        if (txid_equal(rec[o - 1].w, w)) return 0;
    }
    const int r = txid_insert(tab, mask, seed, w, rec[t].state);
    if (r < 0) return -1;
    *added = r;
    return 1;
}

#if defined(__CUDACC__)
// SHA-256(base[a] || base[b]), 32 big-endian bytes; byte by byte (the transactions that need it are rare)
__device__ __forceinline__ void txid_block_sha(const uint8_t* __restrict__ base, Seg a, Seg b, uint8_t out[32])
{
    ShaJob job;
    job.off[0] = a.off; job.len[0] = a.len; job.off[1] = b.off; job.len[1] = b.len; job.off[2] = 0; job.len[2] = 0;
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    const uint64_t total = (uint64_t)a.len + b.len, padded = (total + 9 + 63) / 64 * 64;
    for (uint64_t o = 0; o < padded; o += 64) {
        uint32_t w[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            uint32_t v = 0;
            for (int q = 0; q < 4; q++) v = (v << 8) | sha_msg_byte(base, job, total, padded, o + 4 * k + q);
            w[k] = v;
        }
        sha256_compress(h, w);
    }
    for (int k = 0; k < 8; k++)
        for (int q = 0; q < 4; q++) out[4 * k + q] = (uint8_t)(h[k] >> (24 - 8 * q));
}

// rec[t] = transaction t's id as a table record (state TXID_COMMITTED), or state TXID_EMPTY for none.  env_off: the slot's (begin, end)
// pairs.
__global__ void __launch_bounds__(128)
txid_block_id_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ env_off, uint32_t T, TxidSlot* __restrict__ rec)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    Seg env; env.off = env_off[2 * t]; env.len = env_off[2 * t + 1] - env_off[2 * t];
    uint32_t w[8]; Seg nonce, creator;
    nonce.off = nonce.len = creator.off = creator.len = 0;
    const int k = txid_block_extract(base, env, w, nonce, creator);
    if (k == TXB_COMPUTE) {
        uint8_t d[32];
        txid_block_sha(base, nonce, creator, d);
        txid_words(d, w);
    }
    TxidSlot r;
    for (int q = 0; q < 8; q++) r.w[q] = k == TXB_NONE ? 0u : w[q];
    r.state = k == TXB_NONE ? (uint32_t)TXID_EMPTY : (uint32_t)TXID_COMMITTED;
    rec[t] = r;
}

// count += the ids new to the table
__global__ void __launch_bounds__(256)
txid_block_insert_kernel(TxidSlot* __restrict__ tab, uint32_t mask, uint64_t seed, const TxidSlot* __restrict__ rec, uint32_t T,
                         uint32_t* __restrict__ dd, uint32_t dmask, unsigned long long* __restrict__ count)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    int added = 0;
    txid_block_insert(tab, mask, seed, rec, t, dd, dmask, &added);
    if (added == 1) atomicAdd(count, 1ull);
}
#endif

} }  // namespace fabgpu::bdev
