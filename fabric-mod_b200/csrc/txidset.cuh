// The ledger's committed transaction ids on the device (fabgpu_committed_txids): an open-addressing table in HBM that decide_tx probes
// for checkTxIdDupsLedger (core/committer/txvalidator/v20/validator.go:363-372,462-491; v14/validator.go:334-345).  Host+device code,
// included by blockdev.cuh; the tests' host build runs the same insert and lookup.
//
// A slot is the id's 32 binary bytes (the SHA-256 digest whose lowercase hex is the canonical ChannelHeader.tx_id) and a state.  The slot
// count is a power of two and the library keeps the load at or below 1/2, so every probe chain ends at an empty slot.  The first slot
// probed is a seeded mix of all 32 bytes: ids are caller-chosen strings (a transaction flagged BAD_PROPOSAL_TXID is indexed under the id it
// claimed), and an index taken from the raw bytes would let a submitter line up ids into one long chain that every later lookup walks.
#pragma once

namespace fabgpu { namespace bdev {

enum : uint32_t {
    TXID_EMPTY = 0,
    TXID_CLAIMED = 1,        // an insert of the running launch owns the slot and is writing the id: probers skip it (a different id)
    TXID_COMMITTED = 2,      // GetTransactionByID finds the id: DUPLICATE_TXID
    TXID_UNANSWERABLE = 3    // indexed, but GetTransactionByID fails (an id imported from a snapshot): NOT_VALIDATED
};

struct TxidSlot { uint32_t w[8]; uint32_t state; };

// What block_decide_kernel reads.  broken: a failed call lost ids; every lookup is TXID_UNANSWERABLE until the set is replaced.
struct TxidSetDev {
    const TxidSlot* slots;
    uint32_t mask;           // slot count - 1
    uint32_t broken;
    uint64_t seed;
};

// 32 bytes -> 8 words, little-endian whatever the byte array's alignment
BD_HD void txid_words(const uint8_t* b, uint32_t w[8])
{
    for (int k = 0; k < 8; k++)
        w[k] = (uint32_t)b[4 * k] | ((uint32_t)b[4 * k + 1] << 8) | ((uint32_t)b[4 * k + 2] << 16) | ((uint32_t)b[4 * k + 3] << 24);
}

BD_HD uint64_t txid_mix(const uint32_t w[8], uint64_t seed)
{
    uint64_t h = seed;
    for (int k = 0; k < 4; k++) {
        h ^= (uint64_t)w[2 * k] | ((uint64_t)w[2 * k + 1] << 32);
        h += seed;
        h *= 0xff51afd7ed558ccdull; h ^= h >> 33;
    }
    h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 29;
    return h;
}

BD_HD bool txid_equal(const uint32_t* a, const uint32_t* b)
{
    uint32_t d = 0;
    for (int k = 0; k < 8; k++) d |= a[k] ^ b[k];
    return d == 0;
}

// The slot's state, read so that a published state is seen only with the id written before it
BD_HD uint32_t txid_state_acquire(const TxidSlot* s)
{
#if defined(__CUDA_ARCH__)
    const uint32_t st = *reinterpret_cast<const volatile uint32_t*>(&s->state);
    __threadfence();
    return st;
#else
    return __atomic_load_n(&s->state, __ATOMIC_ACQUIRE);
#endif
}

// Inserts one id with state TXID_COMMITTED or TXID_UNANSWERABLE, or raises the state of the id already held (the larger state wins).
// Two inserts running at the same time must carry different ids (the library removes duplicates within a call): a slot another insert has
// claimed but not yet published is then never this id.  Returns 1 when the id is new, 0 when it was held, -1 when no slot is free.
BD_HD int txid_insert(TxidSlot* tab, uint32_t mask, uint64_t seed, const uint32_t w[8], uint32_t state)
{
    uint32_t pos = (uint32_t)txid_mix(w, seed) & mask;
    for (uint64_t n = 0; n <= (uint64_t)mask; n++, pos = (pos + 1) & mask) {
        TxidSlot* s = tab + pos;
        uint32_t st = txid_state_acquire(s);
        if (st == TXID_EMPTY) {
#if defined(__CUDA_ARCH__)
            st = atomicCAS(&s->state, (uint32_t)TXID_EMPTY, (uint32_t)TXID_CLAIMED);
#else
            __atomic_compare_exchange_n(&s->state, &st, (uint32_t)TXID_CLAIMED, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
#endif
            if (st == TXID_EMPTY) {
                for (int k = 0; k < 8; k++) s->w[k] = w[k];
#if defined(__CUDA_ARCH__)
                __threadfence();
                atomicExch(&s->state, state);
#else
                __atomic_store_n(&s->state, state, __ATOMIC_RELEASE);
#endif
                return 1;
            }
#if defined(__CUDA_ARCH__)
            if (st != TXID_CLAIMED) __threadfence();
#endif
        }
        if (st == TXID_CLAIMED) continue;
        if (txid_equal(s->w, w)) {
            if (state > st) {
#if defined(__CUDA_ARCH__)
                atomicMax(&s->state, state);
#else
                __atomic_store_n(&s->state, state, __ATOMIC_RELEASE);
#endif
            }
            return 0;
        }
    }
    return -1;
}

// The state of `id` (32 bytes): TXID_EMPTY when the set does not hold it.  No insert runs while blocks read the table.
BD_HD uint32_t txid_lookup(const TxidSetDev& set, const uint8_t* id)
{
    if (set.broken) return TXID_UNANSWERABLE;
    uint32_t w[8];
    txid_words(id, w);
    uint32_t pos = (uint32_t)txid_mix(w, set.seed) & set.mask;
    for (uint64_t n = 0; n <= (uint64_t)set.mask; n++, pos = (pos + 1) & set.mask) {
        const TxidSlot& s = set.slots[pos];
        const uint32_t st = s.state;
        if (st == TXID_EMPTY) return TXID_EMPTY;
        if (st != TXID_CLAIMED && txid_equal(s.w, w)) return st;
    }
    return TXID_EMPTY;
}

} }  // namespace fabgpu::bdev
