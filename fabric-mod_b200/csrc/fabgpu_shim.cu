// C-ABI shim of libfabgpu_ecdsa.so (declared in include/fabgpu_ecdsa.h): context, pinned SoA slots, multi-device
// batch split, kernel launches.  No CPU verification fallback lives here by design: a failure is reported to the
// caller, who falls back to the reference's software provider (SURVEY.md section 5).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/fabgpu_ecdsa.h"
#include "bccsp_host.hpp"
#include "blockval.hpp"
#include "capability.hpp"
#include "cuda_owned.hpp"
#include "sha256.cuh"
#include "blockdev_kernels.cuh"
#include "txidblock.cuh"
#include "keypolicy.hpp"
#include "txidset.hpp"
#include "stateset.hpp"
#include "couchval.cuh"
#include "updates.cuh"
#include "pvtdata.cuh"
#include "pvtupdates.cuh"
#include "updatebytes.cuh"
#include "msptable.hpp"
#include "unknownids.cuh"
#include "ecdsa_kernels.cuh"

#if defined(__SSE2__)
#include <emmintrin.h>
#endif

using namespace fabgpu;

namespace {

std::string g_init_error = "";

struct DevSlot {
    Stream stream;
    DevArray<uint8_t> d_in[5];      // qx qy e r s
    DevArray<uint32_t> d_mask;
    DevArray<uint32_t> d_off;
    DevArray<int32_t> d_key_slot;
    DevArray<uint32_t> d_idx;       // dev_cap + 2 words: compaction scratch of mixed batches
    DevArray<uint4> d_scal;         // 4 x dev_cap: scalars u1, u2 of the key-table kernel (ecdsa_prep_kernel)
};

// The point tables of one device, shared by every context of a group (KeyTables).  Members go in reverse order of declaration, with
// this device current (~DevTables).
struct DevTables {
    int id = 0;
    DevArray<aff> gtab;
    DevArray<aff> qtab;       // key_slots tables of FAB_G_WINDOWS * FAB_G_ENTRIES points (per-key fixed-base tables)
    // small key tables (FAB_S_POINTS points each): the pool, the build scratch (grown on demand) and the build stream.  Every
    // enqueue that may read a small table first makes its stream wait for s_ev (the last build): builds are ordered among
    // themselves by s_stream, so one event covers all earlier ones.  The scratch holds s_cap() keys; s_bases is grown last.
    DevArray<aff> stab;
    DevArray<uint8_t> s_keys; DevArray<int32_t> s_slots; DevArray<aff> s_bases;
    size_t s_cap() const { return s_bases.bytes() / (FAB_S_WINDOWS * sizeof(aff)); }
    Stream s_stream; Event s_ev; bool s_ev_set = false;
    ~DevTables() { cudaSetDevice(id); }
};

// What does not depend on the channel: the device tables and the key caches that map keys to them.  fabgpu_init makes a group of one
// context, fabgpu_init_shared adds a context to it; the last context of the group to go frees this.
//
// Locks, in this order (a path may skip any, never reverse two, and never holds one context's lock while taking another's):
//   tab_mu (shared / exclusive) -> a context's fabgpu_ctx::mu -> mu.
// Whoever turns handles into raw slot numbers and then enqueues kernels that read those slots' tables holds tab_mu SHARED from the
// resolution to the last enqueue, in whichever context it enqueues.  fabgpu_keys_register and the small tier hold it EXCLUSIVE while
// they recycle slots (after draining every stream of the device), so no context of the group sits between "resolved" and
// "enqueued" when a slot changes hands.  The maps, slot owners, generations, the free list, the build counters, s_ev / s_ev_set
// and the table contents change only under tab_mu exclusive AND mu; the LRU ticks and the seen counters change under mu (with
// tab_mu shared or exclusive).  A reader holds mu, or tab_mu for what changes only under it exclusively.
struct KeyTables {
    std::vector<DevTables> devs;           // the group's devices, in the contexts' device order
    std::shared_mutex tab_mu;
    std::mutex mu;
    // per-key table cache (fabgpu_keys_register): 64-byte X||Y -> slot, least-recently-used eviction
    int key_slots = 0;
    std::unordered_map<std::string, int> key_map;
    std::vector<std::string> slot_key;
    std::vector<unsigned long long> slot_tick;
    std::vector<uint32_t> slot_gen;          // bumped whenever a slot is recycled: handles carry the generation they were issued under
    unsigned long long tick = 0;
    int key_min_uses = 256;
    // small-table cache (fabgpu_keys_register_small): same protocol as the big tables, least-recently-used eviction in bulk.  A small
    // handle is -2 - ((generation & 0x3ff) << 20 | slot); on the device the code is -2 - slot.
    int small_slots = 0;
    // Cumulative signatures of a key (over all calls) before it earns a small table; < 0: tier off.  A table costs about as much GPU time as a few dozen
    // generic verifications and saves most of one per later signature: 32 is the rent-or-buy point -- by then the key has cost as much on the
    // generic kernel as its table does, so building is at most twice the optimum whatever the key does next, and a block full of one-off keys is
    // not slowed down by thousands of useless builds.
    int small_min_uses = 32;
    struct Key64 { uint8_t b[64]; bool operator==(const Key64& o) const { return memcmp(b, o.b, 64) == 0; } };
    struct Key64Hash { size_t operator()(const Key64& k) const { uint64_t h; memcpy(&h, k.b + 8, 8); return (size_t)(h * 0x9E3779B97F4A7C15ull); } };
    std::unordered_map<Key64, int, Key64Hash> small_map;
    std::vector<Key64> small_key; std::vector<char> small_used;
    std::vector<unsigned long long> small_tick;
    std::vector<uint32_t> small_gen;
    std::vector<int> small_free;
    unsigned long long small_built = 0, small_recycled = 0;     // fabgpu_key_table_stats
    // Keys without any table: signatures seen so far.  Buckets of four (tag, count) entries indexed by a hash of the key bytes -- no allocation
    // on the batch path; a full bucket gives up its least used entry, which only delays that key's table (resolve_key_tables).
    std::vector<uint64_t> seen_tag; std::vector<uint32_t> seen_cnt;
};

// A context's own part of a device.  Members go in reverse order of declaration, with this device current (~Device).
struct Device {
    int id = 0;
    DevTables* tab = nullptr;  // the group's tables on this device
    int sms = 132;            // multiprocessors (launch shapes; read from the device at fabgpu_init)
    DevSlot slot[FABGPU_SLOTS];
    // Stream-ordered scratch for launches on a caller's stream (fabgpu_verify_p256_device_keyed*), which own no slot: allocated and
    // freed in the launch's stream order, so concurrent callers on different streams never share a buffer and never wait for
    // each other.  The pool keeps what it was given (release threshold: no limit) and reuses a block on another stream only when
    // its free has already completed (no dependencies inserted between streams).
    MemPool scal_pool;
    // bitmask exchange over peer memory (fabgpu_peer_mask_*): this rank's receive buffer, the peers' mapped ones (none for this rank:
    // its segment is `local`).  `mapped` comes last so that the mappings are closed before `local` is freed.
    struct Peer {
        DevArray<uint32_t> local; DevArray<uint32_t> done; uint32_t* timeout = nullptr; HostArray<uint32_t> h_timeout;
        int world = 0, rank = 0; size_t words_per_rank = 0; bool ready = false;
        IpcMapping<uint32_t> mapped[FAB_PEER_MAX];
        uint32_t* buf(int p) const { return p == rank ? local.get() : mapped[p].get(); }
    } peer;
    ~Device() { cudaSetDevice(id); }
};

struct HostSlot {
    HostArray<uint8_t> h_in[5];
    HostArray<uint32_t> h_mask;
    HostArray<uint32_t> h_off;
    HostArray<int32_t> h_key_slot;
};

// A device array of the MSP table (fabgpu_ctx::DevMsp), allocated and freed in stream order on the MSP stream (fabgpu_ctx::MspAdmit):
// fabgpu_msp_identities_add grows it while blocks in flight still read the old one -- those keep the pointer they were launched with,
// and the free runs after them (msp_grow).  The destructor's cudaFree runs once every reader has finished (the context is drained).
template <typename T>
struct MspArr {
    T* p = nullptr; size_t cap = 0;
    MspArr() = default;
    MspArr(MspArr&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    MspArr& operator=(MspArr&& o) noexcept
    {
        if (this != &o) { if (p) cudaFree(p); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); }
        return *this;
    }
    ~MspArr() { if (p) cudaFree(p); }
    T* get() const { return p; }
    size_t bytes() const { return cap; }
    void drop(cudaStream_t st) { if (p) cudaFreeAsync(p, st); p = nullptr; cap = 0; }
};

}  // namespace

// Minimal fork-join pool for the host gates (DER parse + packing is ~40 ns/signature single-threaded, which would
// otherwise cap the end-to-end rate near 20 M/s).
class GatePool {
public:
    explicit GatePool(int n) : n_(n < 1 ? 1 : n) {
        for (int t = 1; t < n_; t++) th_.emplace_back([this, t] { loop(t); });
    }
    ~GatePool() {
        { std::lock_guard<std::mutex> lk(mu_); stop_ = true; gen_.fetch_add(1); }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    int size() const { return n_; }
    // runs fn(tid) for tid in [0, size) and returns when all are done
    void run(const std::function<void(int)>& fn) {
        if (n_ == 1) { fn(0); return; }
        { std::lock_guard<std::mutex> lk(mu_); fn_ = &fn; pending_.store(n_ - 1); gen_.fetch_add(1); }
        cv_.notify_all();
        fn(0);
        for (int spin = 0; spin < 20000 && pending_.load(std::memory_order_acquire) != 0; spin++) cpu_relax();
        if (pending_.load(std::memory_order_acquire) == 0) return;
        std::unique_lock<std::mutex> lk(mu_);
        done_.wait(lk, [this] { return pending_.load() == 0; });
    }
private:
    static void cpu_relax() {
#if defined(__SSE2__)
        _mm_pause();
#endif
    }
    // Workers spin briefly for the next job (back-to-back batches arrive within microseconds) before sleeping.
    void loop(int tid) {
        unsigned long long seen = 0;
        for (;;) {
            for (int spin = 0; spin < 20000 && gen_.load(std::memory_order_acquire) == seen; spin++) cpu_relax();
            const std::function<void(int)>* fn;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return gen_.load() != seen; });
                seen = gen_.load();
                if (stop_) return;
                fn = fn_;
            }
            (*fn)(tid);
            if (pending_.fetch_sub(1, std::memory_order_acq_rel) == 1) { std::lock_guard<std::mutex> lk(mu_); done_.notify_one(); }
        }
    }
    int n_;
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    const std::function<void(int)>* fn_ = nullptr;
    std::atomic<int> pending_{0};
    std::atomic<unsigned long long> gen_{0};
    bool stop_ = false;
};

struct fabgpu_ctx {
    std::shared_ptr<KeyTables> kt;     // the group's tables and key caches (first: they go after this context's devices and streams)
    std::vector<Device> devs;
    std::unique_ptr<GatePool> pool;
    HostSlot hslot[FABGPU_SLOTS];
    size_t max_batch = 0;      // per slot, whole context
    size_t dev_cap = 0;        // per device per slot (multiple of 32)
    std::string last_error;
    std::mutex mu;         // guards this context's enqueue state; lock order: kt->tab_mu, mu, kt->mu (KeyTables)
    std::mutex sync_mu;    // one synchronous fabgpu_bccsp_verify_batch at a time
    std::mutex sync_blk_mu;   // one synchronous fabgpu_validate_block / _envelopes at a time
    std::mutex slot0_mu;   // serialises the composite calls that stage through slot 0's pinned buffers
    std::atomic<unsigned long long> launches{0};
    int small_threads_env = 0;                // FABGPU_SMALL_THREADS: CTA width of ecdsa_verify_small_kernel (0 = by batch size)
    // key-table kernel (FABGPU_CACHED_KERNEL): 0 "jac" = Jacobian chain, one signature per thread (ecdsa_verify_cached_kernel) -- the DEFAULT; the
    // others stay selectable for comparison (tools/kbench.py); 1 "ba" = batch-affine with CTA-shared inversions, 3 "ba2" = batch-affine, two
    // signatures per thread, 2 / 4 "l2" / "l4" = the Jacobian chain split over 2 / 4 lanes.  The alternatives stay selectable: they are the measurements.
    int cached_kernel = 0;
    double timing[4] = {0, 0, 0, 0};   // last fabgpu_bccsp_verify_batch: key lookup, host gates, device (H2D+kernel+D2H), scatter [us]
    // block validation (fabgpu_msp_configure / fabgpu_validate_block), device 0 of the context
    blockval::MspTable msp;
    std::vector<blockval::PolicyNode> policy;
    std::vector<std::string> principals;
    std::string channel;
    std::vector<int32_t> identity_slot;
    // per identity: the key tier its table handle was issued in, and is re-issued in when recycled -- TIER_WINDOW (fabgpu_keys_register)
    // or TIER_SMALL (msp_small_tier)
    std::vector<uint8_t> identity_tier;
    struct BlockBufs {
        DevArray<uint8_t> d_block;
        HostArray<uint8_t> h_block;                               // optional pinned staging the caller may fill directly
    } bbs[FABGPU_SLOTS];
    double block_timing[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // host phases [0..4] (see fabgpu_block_timing), device stages [5..9]
    // device-side copy of the MSP view / policy (block_plan_kernel, block_decide_kernel)
    // The identity arrays and the index are MspArr: grown by fabgpu_msp_identities_add with blocks in flight (capacity doubling).
    struct DevMsp {
        MspArr<uint8_t> id_blob, valid, keys_xy; DevArray<uint8_t> channel;
        MspArr<uint32_t> id_off; MspArr<int32_t> key_slot, msp_code, ht_idx; DevArray<int32_t> nodes, principal_code;
        MspArr<int32_t> group;                                        // de-duplication groups (fabgpu_msp_identity_groups), null = identity index
        bool configured = false;                                      // fabgpu_msp_configure installed this table
        msptab::Mirror mirror;                                        // host copy of id_blob / id_off / ht_hash / ht_idx
        std::unordered_map<std::string, int32_t> codes;               // MSP id -> msp_code, identities and principals alike
        DevArray<uint8_t> ns_blob; DevArray<uint32_t> ns_off; DevArray<int32_t> ns_root; int32_t n_ns = 0;    // fabgpu_namespace_policies
        std::vector<int32_t> ns_root_host;                            // the same roots, for the v1.3 mode's ImplicitMeta check
        uint8_t mode = BD_MODE_V20;                       // fabgpu_channel_capability
        DevArray<uint8_t> ver_blob; DevArray<uint32_t> ver_off;       // fabgpu_namespace_versions, null = none
        MspArr<uint32_t> pbits; int32_t pbits_words = 0;              // fabgpu_msp_principal_bits, null = MSP-id member matching
        DevArray<uint8_t> cp_ns_blob, cp_name_blob; DevArray<uint32_t> cp_ns_off, cp_name_off;   // fabgpu_collection_policies, cp_size = 0: none
        DevArray<int32_t> cp_root, cp_idx; DevArray<uint64_t> cp_hash; uint32_t cp_size = 0;
        // fabgpu_key_policies: slots, entry bytes, and the table's nodes after the configured ones in `nodes`; kp_size = 0: none.
        // kp_idx / kp_val stage the changed slots of an update.
        DevArray<bdev::KpSlot> kp_slots, kp_val; DevArray<uint8_t> kp_blob; DevArray<uint32_t> kp_idx; uint32_t kp_size = 0; int32_t kp_n_nodes = 0;
        bool nodes_lost = false;                                      // a failed key-table call lost the configured nodes: no blocks
        MspArr<uint64_t> ht_hash; uint32_t ht_size = 0; int32_t n_ids = 0, n_nodes = 0, n_principals = 0; uint32_t channel_len = 0;
        bool all_slots = true; int classes = 0;                    // which non-big classes the identities' keys fall in (CLASS_*)
    } dm;
    // fabgpu_msp_identities_add: the MSP stream (every DevMsp identity array is allocated, copied and freed on it) and the ordering of
    // admissions, as for the committed tx-id set.  An add runs on `stream` under slot0_mu: it first waits for every slot's last
    // block_decide_kernel (TxidSet::decide_ev, shared) -- blocks submitted before it never see it -- and records `ev`, which every later
    // block_submit makes its first block_resolve_kernel wait for.  The pinned staging buffers rotate, each guarded by its own event, so the
    // host never waits for an add.  `admitted`: an identity was added since the last fabgpu_msp_configure (submits then record decide_ev).
    struct MspAdmit {
        static constexpr int RING = 4;
        Stream stream; Event ev; bool ev_set = false, admitted = false;
        HostArray<uint8_t> h_stage[RING]; Event stage_ev[RING]; bool stage_set[RING] = {}; unsigned seq = 0;
    } adm;
    // fabgpu_block_unknown_identities of a slot's block (unknownids.cuh), on the slot's stream under blk_mu[slot]
    struct UkBufs {
        DevArray<uint64_t> d_hash; DevArray<uint32_t> d_index, d_rep, d_cnt, d_out; DevArray<unsigned long long> d_first;
        HostArray<uint32_t> h_cnt, h_out;
    } uk[FABGPU_SLOTS];
    bdev::KeyPolicyTable kpt;                                      // host mirror of the key policy table
    std::atomic<uint32_t> kl_hint{BD_WRITES_HINT};                 // write records per transaction the block slots are sized for; grows on overflow
    struct GateBufs {                          // fabgpu_bccsp_verify_batch with device-side gates
        // Four groups, each grown together (gate_bufs_reserve).  A group's capacity is read from the array it grows last: signatures
        // (n_cap), signature and digest bytes, keys.
        HostArray<uint8_t> h_sigs, h_digs, h_keys, h_status; HostArray<uint32_t> h_sig_off, h_dig_off; HostArray<int32_t> h_kidx, h_slot_of;
        DevArray<uint8_t> d_sigs, d_digs, d_keys, d_status, d_pre, d_r, d_s, d_e, d_qx, d_qy; DevArray<uint32_t> d_sig_off, d_dig_off, d_mask, d_off;
        DevArray<int32_t> d_kidx, d_slot_of, d_ks; DevArray<uint32_t> d_idx; DevArray<uint4> d_scal;
        size_t n_cap() const { return d_scal.bytes() / 64; }
        size_t sig_cap() const { return d_sigs.bytes(); }
        size_t dig_cap() const { return d_digs.bytes(); }
        size_t k_cap() const { return d_slot_of.bytes() / 4; }
        // fabgpu_bccsp_verify_batch_async .. _wait: what is in flight on this slot
        bool busy = false; bool on_device = false; size_t n = 0;
        std::vector<uint8_t> done_status;       // statuses of a batch that could not take the device-gate path (finished at submit time)
        std::chrono::steady_clock::time_point t_submit;
    } gb[FABGPU_SLOTS];
    std::mutex gb_mu[FABGPU_SLOTS];
    struct DevBlock {
        // grown together in block_submit; the capacity in transactions is read from h_flags, which is grown last
        DevArray<uint32_t> d_env_off; DevArray<bdev::TxDev> d_txs; DevArray<bdev::RawJob> d_raw; DevArray<bdev::ShaJobD> d_sha; DevArray<uint8_t> d_r, d_s, d_qx,
        d_qy, d_gate, d_dig, d_flags; DevArray<int32_t> d_ks, d_ident; DevArray<uint32_t> d_mask, d_off, d_counter, d_idx; DevArray<uint64_t> d_hash;
        DevArray<bdev::Seg> d_seg; DevArray<uint4> d_scal;
        HostArray<uint64_t> h_hash; HostArray<bdev::Seg> h_seg; HostArray<uint32_t> h_counter, h_env_off; HostArray<uint8_t> h_flags;
        size_t tx_cap() const { return h_flags.bytes(); }
        // key policy table installed: write records, the metadata-write set, conflicted transactions (grown together, per block)
        DevArray<bdev::WriteRec> d_w; DevArray<uint64_t> d_md_hash; DevArray<unsigned long long> d_md_min; DevArray<uint32_t> d_md_sum, d_clist; DevArray<uint8_t> d_conf;
        // the block in flight on this slot (fabgpu_validate_*_async .. fabgpu_validate_wait)
        bool busy = false, on_device = false, use_ev = false, kl_on = false, v13 = false; size_t T = 0, W_cap = 0; const uint8_t* block = nullptr;
        bool mvcc_ready = false;                 // fabgpu_validate_wait returned the block and its bytes are still on the device
        bool pvt_ready = false;                  // the same, for fabgpu_validate_pvtdata: fabgpu_validate_mvcc leaves it set
        uint8_t txid_block = 0;                  // fabgpu_committed_txids_add_block: 0 no block submitted, 1 submitted, 2 its ids added
        bool upd_ready = false;                  // fabgpu_validate_mvcc ran on this block (fabgpu_block_updates): cleared by the next submit
        std::vector<uint64_t> dup_keys; std::vector<uint32_t> dup_idx;   // scratch of the duplicate-tx-id pass (per slot: waits may run concurrently)
        std::chrono::steady_clock::time_point t0, t1;
        Event ev[6];                             // created on the first block timed with FABGPU_BLOCK_EVENTS=1
    } dbs[FABGPU_SLOTS];
    std::mutex blk_mu[FABGPU_SLOTS];
    // fabgpu_validate_pvtdata of a slot's block (pvtdata.cuh), on the slot's stream under blk_mu[slot]: pinned staging of the private
    // data, flags and entry tables, and the stage's arrays
    struct PvtBufs {
        HostArray<uint8_t> h_blob, h_flags; HostArray<uint32_t> h_off, h_seq, h_ctr; HostArray<int32_t> h_status; HostArray<unsigned long long> h_verdict;
        DevArray<uint8_t> d_blob, d_flags, d_ent, d_dig; DevArray<uint32_t> d_off, d_seq, d_first, d_n, d_ctr; DevArray<int32_t> d_status;
        DevArray<unsigned long long> d_verdict; DevArray<bdev::PvRec> d_rec; DevArray<bdev::ShaJobP> d_jobs;
        uint32_t rec_hint = PV_REC_HINT;                                                 // collection records per entry the arrays are sized for
        // fabgpu_block_pvt_updates (pvtupdates.cuh): the private batch, rebuilt by every call after the check above
        DevArray<uint32_t> d_wfirst, d_mfirst, d_tbase, d_pctr, d_rmark, d_mark, d_okey, d_out; DevArray<bdev::PuItem> d_item, d_meta;
        DevArray<bdev::ShaJobP> d_mjobs; DevArray<uint8_t> d_mdig; DevArray<bdev::PuKey> d_key; HostArray<uint32_t> h_pctr, h_out;
        uint32_t w_hint = PU_W_HINT, m_hint = PU_M_HINT;                                // writes / metadata writes per entry
    } pvt[FABGPU_SLOTS];
    // fabgpu_committed_txids: the ledger's tx ids on device 0 (txidset.cuh); ledger state, so fabgpu_msp_configure keeps it.  A mutation runs
    // on `stream` under slot0_mu: it first waits for every slot's last block_decide_kernel (decide_ev) -- blocks submitted before it never
    // see it -- and records `ev`, which every later block_submit makes its decide stage wait for.  The host never waits for an add (that
    // would wait for the decide stage of the block just submitted): the pinned staging buffers rotate, each guarded by its own event, and
    // growth is decided on `count` (exact as of the last finished mutation) + `pending` (ids sent since, an upper bound of the new ones).
    struct TxidSet {
        static constexpr int RING = 4;
        Stream stream; Event ev; bool ev_set = false;
        Event decide_ev[FABGPU_SLOTS]; bool decide_set[FABGPU_SLOTS] = {};
        HostArray<bdev::TxidSlot> h_stage[RING]; Event stage_ev[RING]; bool stage_set[RING] = {}; unsigned seq = 0;
        DevArray<bdev::TxidSlot> d_stage;
        HostArray<unsigned long long> h_count; DevArray<unsigned long long> d_count;
        bdev::TxidSlot* table = nullptr; uint64_t slots = 0;                   // table: stream-ordered allocation on `stream`
        const uint64_t seed = txid::random_seed();
        bool installed = false, broken = false; unsigned long long count = 0, pending = 0;
        // fabgpu_committed_txids_add_block: the block's id records and its de-duplication index (one add runs at a time on `stream`);
        // read_ev[slot] follows the last kernel that reads the slot's block and envelope table, and the slot's next submit waits for it
        DevArray<bdev::TxidSlot> d_brec; DevArray<uint32_t> d_dd;
        Event read_ev[FABGPU_SLOTS]; bool read_set[FABGPU_SLOTS] = {};
        ~TxidSet() { if (table) cudaFree(table); }
    } txid;
    // fabgpu_state_versions: the world state's key versions on device 0 (stateset.cuh); ledger state, so fabgpu_msp_configure keeps it.
    // Every call runs under slot0_mu and returns with its stream synchronised -- replace and update on `stream`, fabgpu_validate_mvcc on
    // the slot's stream -- so `count` is exact between calls and growth is decided on it plus the keys one call may add.  Blocks in
    // flight never read the table.
    struct StateSet {
        Stream stream;
        HostArray<bdev::StateSlot> h_stage; DevArray<bdev::StateSlot> d_stage;
        HostArray<unsigned long long> h_count; DevArray<unsigned long long> d_count;   // [0..2]: StateSetDev::count, [3]: a failed upsert
        bdev::StateSlot* table = nullptr; uint64_t slots = 0;                            // stream-ordered allocation
        const uint64_t seed = txid::random_seed();
        bool installed = false, broken = false, open = false; uint64_t height = 0; unsigned long long count[3] = {0, 0, 0};
        // the MVCC stage's arrays (one stage runs at a time)
        DevArray<bdev::MvccRec> d_rec; DevArray<uint32_t> d_first, d_n, d_mlist, d_ctr; DevArray<uint8_t> d_info, d_tv, d_flags;
        DevArray<bdev::MvccKey> d_key; HostArray<uint8_t> h_flags; HostArray<uint32_t> h_ctr;
        uint32_t rec_hint = 8;                                                           // records per transaction the arrays are sized for
        // the ordered index of the public keys (fabgpu_state_versions_indexed, stateindex.cuh): base and delta runs, the delta's next
        // form, a maintenance step's new run and flags, the key bytes; icnt as StateIndexDev documents, h_icnt its copy after each call
        bool indexed = false;
        DevArray<bdev::IndexEntry> ix_base, ix_delta, ix_delta2, ix_fresh; DevArray<uint8_t> ix_heap; DevArray<uint32_t> ix_flag;
        DevArray<unsigned long long> d_icnt; HostArray<unsigned long long> h_icnt; unsigned long long icnt[5] = {0, 0, 0, 0, 0};
        DevArray<bdev::MvccRange> d_rng; DevArray<bdev::MerkleState> d_mk; DevArray<uint32_t> d_first_rng, d_n_rng; DevArray<bdev::WrittenKey> d_wk, d_wk2, d_cand;
        DevArray<uint8_t> d_cand_bytes;
        uint32_t rng_hint = 1;                                                           // range records per transaction
        // the state database the stage restates (fabgpu_state_database); CouchDB adds the key and value pre-pass (couchval.cuh)
        bool couch = false;
        DevArray<bdev::CvWrite> d_cvw; DevArray<uint32_t> d_cv_first, d_cv_n; DevArray<uint8_t> d_cv_undet, d_cv_code; DevArray<uint32_t> d_cv_long;
        uint32_t cv_hint = 4;                                                            // public writes per transaction
        // fabgpu_block_updates of the block the stage last ran on (updates.cuh), built by the first call from the stage's arrays, which
        // stay untouched until the next stage.  upd_slot -1: none (the next stage or state call clears it).  upd_incomplete: open, broken
        // or aliased as the stage left it, or found so by the build.
        int upd_slot = -1; uint64_t upd_block = 0; uint32_t upd_R = 0, upd_K = 0, upd_T = 0; bool upd_incomplete = false, upd_built = false;
        size_t upd_n[2] = {0, 0};
        std::vector<uint8_t> upd_flags;                                                  // the final flags the stage returned (fabgpu_block_pvt_updates)
        DevArray<bdev::UdPair> d_upair; DevArray<bdev::UdKey> d_ukey; DevArray<bdev::UdSeg> d_useg; DevArray<uint8_t> d_uneed, d_utxneed, d_umeta;
        DevArray<uint32_t> d_ubase, d_umark, d_uokey, d_uomoff, d_uout, d_uctr; HostArray<uint32_t> h_uctr;
        // fabgpu_block_update_bytes (updatebytes.cuh): the batch's records sorted by (namespace, collection, key) -- in d_bitem or, when
        // upd_sorted, d_bitem2 -- and each record's index among the COMMITTED-value records (upd_ncom of them), built by the first call
        // for the batch; then per call the committed values, the KVWrites' offsets and chunks, and the bytes
        bool upd_ordered = false; int upd_sorted = 0; uint32_t upd_ncom = 0;
        DevArray<bdev::UbItem> d_bitem, d_bitem2; DevArray<uint32_t> d_bcidx, d_bchunk, d_bvoff, d_bctr; DevArray<unsigned long long> d_boff;
        DevArray<uint8_t> d_bval, d_bout; HostArray<uint32_t> h_bctr; HostArray<unsigned long long> h_btot;
        ~StateSet() { if (table) cudaFree(table); }
    } sv;
    // The members above go in reverse order of declaration -- block slots and MSP copy first, then devices, then the group's tables if
    // this context was the last to hold them -- with device 0 current.
    ~fabgpu_ctx() { if (!devs.empty()) cudaSetDevice(devs[0].id); }
};

namespace {

#define CK(ctx, call)                                                                                       \
    do {                                                                                                    \
        cudaError_t e_ = (call);                                                                            \
        if (e_ != cudaSuccess) {                                                                            \
            char buf_[512];                                                                                 \
            snprintf(buf_, sizeof buf_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            if (ctx) (ctx)->last_error = buf_; else g_init_error = buf_;                                    \
            return FABGPU_E_CUDA;                                                                           \
        }                                                                                                   \
    } while (0)

// Reserves arrays in order (CudaArray::reserve) until one fails; the arrays after that one are freed instead.  A group whose capacity is
// read from the array it grows last therefore reads as empty after a failed grow, and the next call grows the whole group again.
struct Grow {
    fabgpu_ctx* ctx;
    int rc = FABGPU_OK;
    template <typename A> void operator()(A& a, size_t bytes) { if (rc == FABGPU_OK) rc = a.reserve(ctx, bytes); else a = A(); }
};

// Makes `a` hold at least `need` bytes (plus 8 of slack: word-wise readers may touch the aligned word past the end), keeping its first
// `keep` bytes: a larger array (at least twice the old capacity) is allocated and copied in stream order on st.  The old array is freed
// there too, or, with `retire`, handed over to be freed later (after the stream has waited for the blocks that still read it).
// fresh: reallocate even when the array is large enough.
template <typename T>
static int msp_grow(fabgpu_ctx* ctx, MspArr<T>& a, cudaStream_t st, size_t need, size_t keep, std::vector<void*>* retire = nullptr,
                    bool fresh = false)
{
    need += 8;
    if (need <= a.cap && !fresh) return FABGPU_OK;
    const size_t cap = std::max(need, 2 * a.cap);
    void* p = nullptr;
    CK(ctx, cudaMallocAsync(&p, cap, st));
    if (keep && cudaMemcpyAsync(p, a.p, keep, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        cudaFreeAsync(p, st); ctx->last_error = "MSP table copy failed"; return FABGPU_E_CUDA;
    }
    if (retire) { if (a.p) retire->push_back(a.p); a.p = nullptr; a.cap = 0; }
    else a.drop(st);
    a.p = static_cast<T*>(p); a.cap = cap;
    return FABGPU_OK;
}

bool fault_injected()
{
    const char* v = getenv("FABGPU_FAULT_INJECT");
    return v && v[0] == '1';
}

size_t round_up32(size_t x) { return (x + 31) / 32 * 32; }

// 32-byte copy into a pinned staging buffer with streaming stores: the lines never become dirty in this core's cache,
// so the H2D DMA that follows does not have to snoop 16+ cores across two sockets (measured: that snooping more than
// doubled the copy phase when the gates ran multi-threaded).
inline void stage32(uint8_t* dst, const uint8_t* src)
{
#if defined(__SSE2__)
    const __m128i a = _mm_loadu_si128((const __m128i*)src), b = _mm_loadu_si128((const __m128i*)(src + 16));
    _mm_stream_si128((__m128i*)dst, a);
    _mm_stream_si128((__m128i*)(dst + 16), b);
#else
    memcpy(dst, src, 32);
#endif
}
inline void stage_i32(int32_t* dst, int32_t v)
{
#if defined(__SSE2__)
    _mm_stream_si32((int*)dst, v);
#else
    *dst = v;
#endif
}
// bytes -> pinned staging with streaming stores (16-byte aligned body), see stage32
inline void stage_copy(uint8_t* dst, const uint8_t* src, size_t n)
{
#if defined(__SSE2__)
    size_t i = 0;
    while (i < n && ((uintptr_t)(dst + i) & 15u)) { dst[i] = src[i]; i++; }
    for (; i + 16 <= n; i += 16) _mm_stream_si128((__m128i*)(dst + i), _mm_loadu_si128((const __m128i*)(src + i)));
    for (; i < n; i++) dst[i] = src[i];
#else
    memcpy(dst, src, n);
#endif
}
inline void stage_fence()
{
#if defined(__SSE2__)
    _mm_sfence();
#endif
}

// mode: 0 = no signature has a key table (generic kernel only), 1 = all have one (cached kernel only),
//       2 = mixed (cached kernel, then the generic kernel fills in the rest)
//       3 = all have a SMALL table (key_slot codes <= -2 throughout)
// In mode 2 key_slot codes decide per signature: >= 0 big table, -1 none, <= -2 small table (see compact_classes_kernel).
enum { MODE_GENERIC = 0, MODE_CACHED = 1, MODE_MIXED = 2, MODE_SMALL = 3 };

// CTA width of the small-table kernel: as for the key-table kernel, a batch that fits one wave of 512-thread CTAs runs best as such; when
// the count is only an upper bound (compacted list) small CTAs spread the unknown number of live warps over all SMs.  FABGPU_SMALL_THREADS
// overrides (measurements).
unsigned small_threads(const fabgpu_ctx* ctx, const Device& dv, size_t n, bool bound_only)
{
    if (ctx->small_threads_env) return (unsigned)ctx->small_threads_env;
    if (bound_only) return 128;
    const size_t sms = (size_t)dv.sms;
    if (n > sms * 384) return (n <= sms * FAB_SMALL_THREADS) ? FAB_SMALL_THREADS : 256;
    return 128;
}
// classes (mode 2 with scratch): which of the non-big classes the batch may contain -- a class the caller knows to be absent is not launched.
enum { CLASS_SMALL = 1, CLASS_GENERIC = 2 };
enum : uint8_t { TIER_WINDOW = 0, TIER_SMALL = 1 };    // fabgpu_ctx::identity_tier
// n_dev / n_base (block path): the batch is [0, min(n, n_base + *n_dev)) with *n_dev written by an earlier kernel of the stream.
int launch_verify(fabgpu_ctx* ctx, const Device& dv, int mode, const int32_t* key_slot, const uint8_t* qx, const uint8_t* qy,
                  const uint8_t* e, const uint8_t* r, const uint8_t* s, size_t n, uint32_t* mask, uint32_t* off, cudaStream_t st,
                  const uint32_t* n_dev = nullptr, uint32_t n_base = 0, const PeerOut* peer = nullptr, uint32_t* scratch_idx = nullptr,
                  int classes = CLASS_SMALL | CLASS_GENERIC, uint4* scal = nullptr)
{
    PeerOut po; memset(&po, 0, sizeof po);
    const bool fused_peer = peer && mode == MODE_CACHED && (ctx->cached_kernel == 0 || ctx->cached_kernel == 1 || ctx->cached_kernel == 3) && n > 0 && !n_dev;
    if (fused_peer) po = *peer;
    if (peer && !fused_peer) {                            // several kernels write the mask: scatter it afterwards (below)
        if (n_dev) { ctx->last_error = "peer exchange needs a host-known batch size"; return FABGPU_E_ARG; }
    }
    if (n == 0 && !peer) return FABGPU_OK;
    if ((mode == MODE_MIXED || mode == MODE_SMALL) && dv.tab->s_ev_set) CK(ctx, cudaStreamWaitEvent(st, dv.tab->s_ev.get(), 0));   // small tables still being built
    if (mode == MODE_SMALL && n > 0) {
        const unsigned sthreads = small_threads(ctx, dv, n, false);
        ecdsa_verify_small_kernel<<<(unsigned)((n + sthreads - 1) / sthreads), sthreads, 0, st>>>(
            nullptr, nullptr, 0u, key_slot, e, r, s, (uint32_t)n, dv.tab->gtab.get(), dv.tab->stab.get(), mask, off);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    if (mode != MODE_GENERIC && mode != MODE_SMALL && n > 0) {
        // CTA shape (the kernel allows up to FAB_CACHED_THREADS = 512 threads at 128 registers, i.e. one such CTA per SM).
        // A batch that fits one wave of 512-thread CTAs (64k: 128 CTAs on 132 SMs) runs fastest as such, ahead of 512 CTAs of
        // 128 threads; beyond one wave 256-thread CTAs quantise best; below ~12 warps per SM small CTAs spread over all SMs win
        // (fewer warps per scheduler = lower latency per warp), and so they do when the batch size is only an upper bound.
        if (ctx->cached_kernel == 2 || ctx->cached_kernel == 4) {
            // lane-split Jacobian chain (measurement variant): 2 or 4 lanes per signature
            const unsigned sigs = FAB_LANES_THREADS / (unsigned)ctx->cached_kernel, blocks = (unsigned)((n + sigs - 1) / sigs);
            uint32_t nn = (uint32_t)n;
            if (n_dev) { ctx->last_error = "the lane-split kernel has no device-side batch size"; return FABGPU_E_ARG; }
            if (ctx->cached_kernel == 2) ecdsa_verify_lanes_kernel<2><<<blocks, FAB_LANES_THREADS, 0, st>>>(key_slot, e, r, s, nn, dv.tab->gtab.get(), dv.tab->qtab.get(), mask, off);
            else ecdsa_verify_lanes_kernel<4><<<blocks, FAB_LANES_THREADS, 0, st>>>(key_slot, e, r, s, nn, dv.tab->gtab.get(), dv.tab->qtab.get(), mask, off);
        } else if (ctx->cached_kernel == 3 && !n_dev && !fused_peer) {
            // batch-affine, two signatures per thread, no CTA exchange
            const unsigned per = 2 * FAB_BA2_THREADS, blocks = (unsigned)((n + per - 1) / per);
            ecdsa_verify_ba2_kernel<<<blocks, FAB_BA2_THREADS, 0, st>>>(key_slot, e, r, s, (uint32_t)n, dv.tab->gtab.get(), dv.tab->qtab.get(), mask, off);
        } else if (ctx->cached_kernel == 1 || ctx->cached_kernel == 3) {
            // batch-affine accumulation with CTA-shared inversions (ecdsa_batchaffine.cuh): fixed CTA width
            const unsigned blocks = (unsigned)((n + FAB_BA_THREADS - 1) / FAB_BA_THREADS);
            ecdsa_verify_ba_kernel<<<blocks, FAB_BA_THREADS, 0, st>>>(key_slot, e, r, s, (uint32_t)n, dv.tab->gtab.get(), dv.tab->qtab.get(), mask, off, n_dev, n_base, po);
        } else {
        // the scalars (ecdsa_prep_kernel), then the chain.  scal: 64 bytes per signature from the caller's slot, or stream-ordered from
        // the device's pool when the launch has no slot
        const bool own = scal == nullptr;
        if (own) CK(ctx, cudaMallocFromPoolAsync((void**)&scal, 64 * n, dv.scal_pool.get(), st));
        ecdsa_prep_kernel<<<(unsigned)((n + FAB_PREP_THREADS - 1) / FAB_PREP_THREADS), FAB_PREP_THREADS, 0, st>>>(key_slot, e, r, s, (uint32_t)n, scal, n_dev, n_base);
        ctx->launches++;
        unsigned threads = 128;
        const size_t sms = (size_t)dv.sms;
        if (!n_dev && n > sms * 384) threads = (n <= sms * FAB_CACHED_THREADS) ? FAB_CACHED_THREADS : 256;
        const unsigned blocks = (unsigned)((n + threads - 1) / threads);
        ecdsa_verify_cached_kernel<<<blocks, threads, 0, st>>>(key_slot, scal, r, (uint32_t)n, dv.tab->gtab.get(), dv.tab->qtab.get(), mask, off, n_dev, n_base, po);
        if (own) CK(ctx, cudaFreeAsync(scal, st));
        }
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    if (mode == MODE_MIXED && n > 0 && scratch_idx) {
        // signatures without a big table: compact their indices by class, then whole warps of small-table / generic arithmetic
        // (see compact_classes_kernel).  scratch_idx: n + 2 words owned by the caller's slot (indices, then the two counters).
        CK(ctx, cudaMemsetAsync(scratch_idx + n, 0, 8, st));
        compact_classes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(key_slot, (uint32_t)n, scratch_idx, scratch_idx + n, n_dev, n_base);
        if (classes & CLASS_SMALL) {
            const unsigned sthreads = small_threads(ctx, dv, n, true);
            ecdsa_verify_small_kernel<<<(unsigned)((n + sthreads - 1) / sthreads), sthreads, 0, st>>>(
                scratch_idx, scratch_idx + n + 1, (uint32_t)n, key_slot, e, r, s, (uint32_t)n, dv.tab->gtab.get(), dv.tab->stab.get(), mask, off);
        }
        if (classes & CLASS_GENERIC)
            ecdsa_verify_indexed_kernel<<<(unsigned)((n + FAB_INDEXED_THREADS - 1) / FAB_INDEXED_THREADS), FAB_INDEXED_THREADS, 0, st>>>(
                scratch_idx, scratch_idx + n, qx, qy, e, r, s, dv.tab->gtab.get(), mask, off);
        ctx->launches += 1 + ((classes & CLASS_SMALL) ? 1 : 0) + ((classes & CLASS_GENERIC) ? 1 : 0);
        CK(ctx, cudaGetLastError());
    } else if (mode == MODE_MIXED && n > 0) {
        // no scratch (launches on a caller's stream): the generic kernel filters on key_slot itself
        const unsigned gthreads = 128, blocks = (unsigned)((n + gthreads - 1) / gthreads);
        ecdsa_verify_kernel<<<blocks, gthreads, 0, st>>>(key_slot, qx, qy, e, r, s, (uint32_t)n, dv.tab->gtab.get(), mask, off, n_dev, n_base);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    if (mode == MODE_GENERIC && n > 0) {
        // same reasoning for the generic kernel: one wave of 448-thread CTAs when the batch fills it, 256-thread CTAs beyond,
        // 64-thread CTAs for small batches
        unsigned gthreads = 64;
        if (!n_dev && n > (size_t)dv.sms * 192) gthreads = (n <= (size_t)dv.sms * FAB_VERIFY_THREADS) ? FAB_VERIFY_THREADS : 256;
        const unsigned blocks = (unsigned)((n + gthreads - 1) / gthreads);
        ecdsa_verify_kernel<<<blocks, gthreads, 0, st>>>(nullptr, qx, qy, e, r, s, (uint32_t)n, dv.tab->gtab.get(), mask, off, n_dev, n_base);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    if (peer && !fused_peer) {
        const uint32_t words = (uint32_t)((n + 31) / 32);
        peer_scatter_kernel<<<words ? (words + 127) / 128 : 1, 128, 0, st>>>(mask, words, *peer);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    return FABGPU_OK;
}

// (The generation field is 19 bits: a handle kept across 524 288 recyclings of ITS slot would match again.  At one recycling per registration
// call that is days of continuous eviction of one slot while a caller sits on a stale handle; the Go provider re-reads the handle from the key
// object on every batch, so it never holds one that long.)
// A key handle is (generation << 12) | slot.  A handle issued before its slot was recycled no longer matches the slot's
// generation and silently degrades to "no table" (-1): the generic kernel then verifies against the Qx/Qy the caller
// supplied, so a stale handle can cost speed but never correctness.
inline int32_t make_handle(const fabgpu_ctx* ctx, int sl) { return (int32_t)(((ctx->kt->slot_gen[sl] & 0x7ffffu) << 12) | (uint32_t)sl); }
inline int32_t make_small_handle(const fabgpu_ctx* ctx, int sl) { return -2 - (int32_t)(((ctx->kt->small_gen[sl] & 0x3ffu) << 20) | (uint32_t)sl); }
// handle -> device code: >= 0 big-table slot, -2 - slot for a live small table, -1 otherwise (no table, stale handle)
inline int32_t handle_to_slot(const fabgpu_ctx* ctx, int32_t h)
{
    if (h <= -2) {
        const uint32_t v = (uint32_t)(-2 - h);
        const int sl = (int)(v & 0xfffffu);
        if (sl >= ctx->kt->small_slots || (v >> 20) != (ctx->kt->small_gen[sl] & 0x3ffu) || !ctx->kt->small_used[sl]) return -1;
        return -2 - sl;
    }
    if (h < 0) return -1;
    const int sl = h & 0xfff;
    if (sl >= ctx->kt->key_slots || ((uint32_t)h >> 12) != (ctx->kt->slot_gen[sl] & 0x7ffffu) || ctx->kt->slot_key[sl].empty()) return -1;
    return sl;
}

int slots_mode(const int32_t* ks, size_t n, int* classes)
{
    bool any_c = false, any_g = false, any_s = false;
    for (size_t i = 0; i < n; i++) { if (ks[i] >= 0) any_c = true; else if (ks[i] == -1) any_g = true; else any_s = true; }
    *classes = (any_s ? CLASS_SMALL : 0) | (any_g ? CLASS_GENERIC : 0);
    if (!any_c && !any_g && any_s) return MODE_SMALL;
    if (!any_c && !any_s) return MODE_GENERIC;
    return (any_g || any_s) ? MODE_MIXED : MODE_CACHED;
}

int enqueue_slot(fabgpu_ctx* ctx, int slot, size_t n, bool keyed)
{
    // contiguous 32-aligned ranges per device
    const size_t ndev = ctx->devs.size();
    const size_t per = round_up32((n + ndev - 1) / ndev);
    for (size_t d = 0; d < ndev; d++) {
        const size_t begin = std::min(n, d * per), end = std::min(n, (d + 1) * per);
        const size_t cnt = end - begin;
        if (cnt == 0) continue;
        Device& dv = ctx->devs[d];
        DevSlot& ds = dv.slot[slot];
        HostSlot& hs = ctx->hslot[slot];
        CK(ctx, cudaSetDevice(dv.id));
        if (keyed) for (size_t i = begin; i < end; i++) hs.h_key_slot.get()[i] = handle_to_slot(ctx, hs.h_key_slot.get()[i]);   // handles -> live slots
        int classes = CLASS_GENERIC;
        const int mode = keyed ? slots_mode(hs.h_key_slot.get() + begin, cnt, &classes) : MODE_GENERIC;
        for (int a = ((mode == MODE_CACHED || mode == MODE_SMALL) ? 2 : 0); a < 5; a++)     // a range where every key has a table needs no Qx/Qy on the device
            CK(ctx, cudaMemcpyAsync(ds.d_in[a].get(), hs.h_in[a].get() + 32 * begin, 32 * cnt, cudaMemcpyHostToDevice, ds.stream.get()));
        if (mode != MODE_GENERIC)
            CK(ctx, cudaMemcpyAsync(ds.d_key_slot.get(), hs.h_key_slot.get() + begin, 4 * cnt, cudaMemcpyHostToDevice, ds.stream.get()));
        int rc = launch_verify(ctx, dv, mode, ds.d_key_slot.get(), ds.d_in[0].get(), ds.d_in[1].get(), ds.d_in[2].get(), ds.d_in[3].get(), ds.d_in[4].get(), cnt, ds.d_mask.get(),
                               ds.d_off.get(), ds.stream.get(), nullptr, 0, nullptr, ds.d_idx.get(), classes, ds.d_scal.get());
        if (rc) return rc;
        const size_t words = (cnt + 31) / 32;
        CK(ctx, cudaMemcpyAsync(hs.h_mask.get() + begin / 32, ds.d_mask.get(), 4 * words, cudaMemcpyDeviceToHost, ds.stream.get()));
        CK(ctx, cudaMemcpyAsync(hs.h_off.get() + begin / 32, ds.d_off.get(), 4 * words, cudaMemcpyDeviceToHost, ds.stream.get()));
    }
    return FABGPU_OK;
}

int wait_slot(fabgpu_ctx* ctx, int slot)
{
    for (auto& dv : ctx->devs) {
        CK(ctx, cudaSetDevice(dv.id));
        CK(ctx, cudaStreamSynchronize(dv.slot[slot].stream.get()));
    }
    return FABGPU_OK;
}

// with == nullptr: a new group -- the tables are allocated and the generator's is built; otherwise the context joins with's group
// on with's devices and allocates only its own buffers.
int init_impl(fabgpu_ctx* ctx, const int* device_ids, int n_dev, size_t max_batch, const fabgpu_ctx* with = nullptr)
{
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        ctx->last_error = std::string("no usable CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                          " (libfabgpu_ecdsa has no CPU fallback; use the software provider)";
        return FABGPU_E_NO_DEVICE;
    }
    std::vector<int> ids;
    if (with) for (const auto& dv : with->devs) ids.push_back(dv.id);
    else if (device_ids == nullptr || n_dev <= 0) ids.push_back(0);
    else ids.assign(device_ids, device_ids + n_dev);
    for (int id : ids)
        if (id < 0 || id >= count) { ctx->last_error = "device id out of range"; return FABGPU_E_NO_DEVICE; }
    if (max_batch == 0) { ctx->last_error = "max_batch must be > 0"; return FABGPU_E_ARG; }
    ctx->max_batch = max_batch;
    {
        int hw = (int)std::thread::hardware_concurrency();
        const char* ev = getenv("FABGPU_GATE_THREADS");
        int want = ev ? atoi(ev) : std::max(1, std::min(hw > 0 ? hw / 2 : 1, 32));   // gates and block parsing are latency-bound
        ctx->pool.reset(new GatePool(want));
        const char* sth = getenv("FABGPU_SMALL_THREADS");
        if (sth) { const int v = atoi(sth); if (v == 64 || v == 128 || v == 256 || v == 512) ctx->small_threads_env = v; }
        const char* ck = getenv("FABGPU_CACHED_KERNEL");
        if (ck) ctx->cached_kernel = (ck[0] == 'j' || ck[0] == '0') ? 0 : (ck[0] == 'l' ? (ck[1] == '4' ? 4 : 2) : (ck[0] == 'b' && ck[1] == 'a' && ck[2] == '2' ? 3 : 1));   // "jac" / "0": the Jacobian-chain kernel; "l2" / "l4": its lane-split variant
    }
    const bool fresh = with == nullptr;
    if (!fresh) ctx->kt = with->kt;
    else {
        ctx->kt = std::make_shared<KeyTables>();
        ctx->kt->devs = std::vector<DevTables>(ids.size());   // DevTables is not movable: the vector is built at its final size
        // Per-key tables are 64 MiB each (FAB_WQ = 16), per device.  The request (default 256 = 16 GiB of an H100's 80 GB) is
        // capped so that the tables never take more than half of the smallest device's free memory.
        const char* ks = getenv("FABGPU_KEY_SLOTS");
        ctx->kt->key_slots = ks ? std::max(1, atoi(ks)) : 256;
        if (ctx->kt->key_slots > 4096) ctx->kt->key_slots = 4096;     // a handle keeps 12 bits for the slot
        const size_t per_key = (size_t)FAB_Q_WINDOWS * FAB_Q_ENTRIES * sizeof(aff);
        for (int id : ids) {
            size_t free_b = 0, total_b = 0;
            CK(ctx, cudaSetDevice(id));
            CK(ctx, cudaMemGetInfo(&free_b, &total_b));
            // a device listed k times in device_ids holds k sets of tables: each gets a k-th of the room
            const size_t uses = (size_t)std::count(ids.begin(), ids.end(), id);
            const size_t g_bytes = (size_t)FAB_G_WINDOWS * FAB_G_ENTRIES * sizeof(aff);
            const size_t room = free_b > 2 * g_bytes * uses ? (free_b - 2 * g_bytes * uses) / 2 / uses : 0;
            ctx->kt->key_slots = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->kt->key_slots, room / per_key));
        }
        ctx->kt->slot_key.assign(ctx->kt->key_slots, std::string());
        ctx->kt->slot_tick.assign(ctx->kt->key_slots, 0ull);
        ctx->kt->slot_gen.assign(ctx->kt->key_slots, 0u);
        // Small tables (FAB_S_POINTS * 64 bytes = 264 KiB each): default 16 384 of them (4.4 GB); FABGPU_SMALL_SLOTS = 0 turns the tier off.
        const char* ss = getenv("FABGPU_SMALL_SLOTS");
        ctx->kt->small_slots = ss ? std::max(0, atoi(ss)) : 16384;
        if (ctx->kt->small_slots > (1 << 20)) ctx->kt->small_slots = 1 << 20;       // a handle keeps 20 bits for the slot
        for (int id : ids) {
            size_t free_b = 0, total_b = 0;
            CK(ctx, cudaSetDevice(id));
            CK(ctx, cudaMemGetInfo(&free_b, &total_b));
            const size_t per_small = (size_t)FAB_S_POINTS * sizeof(aff);
            const size_t uses = (size_t)std::count(ids.begin(), ids.end(), id);
            ctx->kt->small_slots = (int)std::min<size_t>((size_t)ctx->kt->small_slots, free_b / 8 / uses / per_small);
        }
        ctx->kt->small_key.assign(ctx->kt->small_slots, KeyTables::Key64());
        ctx->kt->small_used.assign(ctx->kt->small_slots, 0);
        ctx->kt->small_tick.assign(ctx->kt->small_slots, 0ull);
        ctx->kt->small_gen.assign(ctx->kt->small_slots, 0u);
        ctx->kt->small_free.clear();
        for (int sl = ctx->kt->small_slots - 1; sl >= 0; sl--) ctx->kt->small_free.push_back(sl);
        ctx->kt->seen_tag.assign((size_t)1 << 18, 0ull); ctx->kt->seen_cnt.assign((size_t)1 << 18, 0u);
        const char* smu = getenv("FABGPU_SMALL_MIN_USES");
        ctx->kt->small_min_uses = smu ? atoi(smu) : 32;
        if (ctx->kt->small_slots == 0) ctx->kt->small_min_uses = -1;
        const char* mu = getenv("FABGPU_KEY_MIN_USES");
        ctx->kt->key_min_uses = mu ? atoi(mu) : 256;           // a table costs about 300 generic verifications to build
    }
    ctx->dev_cap = round_up32((max_batch + ids.size() - 1) / ids.size());
    ctx->devs = std::vector<Device>(ids.size());          // Device is not movable: the vector is built at its final size
    const size_t words = ctx->dev_cap / 32;
    const size_t tab_entries = (size_t)FAB_G_WINDOWS * FAB_G_ENTRIES;
    for (size_t d = 0; d < ids.size(); d++) {
        Device& dv = ctx->devs[d];
        dv.id = ids[d];
        dv.tab = &ctx->kt->devs[d];
        CK(ctx, cudaSetDevice(dv.id));
        CK(ctx, cudaDeviceGetAttribute(&dv.sms, cudaDevAttrMultiProcessorCount, dv.id));
        {   // Table gathers read 64-byte points at random addresses: by default the L2 fetches 128 bytes around a miss (two sectors'
            // worth of DRAM traffic per point).  FABGPU_L2_FETCH = 32 / 64 / 128 sets cudaLimitMaxL2FetchGranularity; default 64.
            const char* fg = getenv("FABGPU_L2_FETCH");
            const size_t want = fg ? (size_t)atoi(fg) : 64;
            if (want == 32 || want == 64 || want == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, want);   // a hint: failure is not an error
            (void)cudaGetLastError();
        }
        Grow grow{ctx};
        cudaStream_t st = nullptr;
        if (fresh) {
            dv.tab->id = dv.id;
            grow(dv.tab->gtab, tab_entries * sizeof(aff));
            grow(dv.tab->qtab, (size_t)ctx->kt->key_slots * FAB_Q_WINDOWS * FAB_Q_ENTRIES * sizeof(aff));
            if (ctx->kt->small_slots > 0) {
                grow(dv.tab->stab, (size_t)ctx->kt->small_slots * FAB_S_POINTS * sizeof(aff));
                // build scratch for up to 16 384 keys per registration, allocated once: growing it later costs a cudaFree + cudaMalloc pair in the
                // middle of traffic (the pair waits for all work in flight)
                const size_t c = (size_t)std::min(ctx->kt->small_slots, 16384);
                grow(dv.tab->s_bases, c * FAB_S_WINDOWS * sizeof(aff));
                grow(dv.tab->s_keys, 64 * c);
                grow(dv.tab->s_slots, 4 * c);
            }
            if (grow.rc) return grow.rc;
            CK(ctx, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
            dv.tab->s_stream.reset(st);
            cudaEvent_t ev = nullptr;
            CK(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            dv.tab->s_ev.reset(ev);
        }
        for (auto& ds : dv.slot) {
            CK(ctx, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
            ds.stream.reset(st);
            for (auto& p : ds.d_in) grow(p, 32 * ctx->dev_cap);
            grow(ds.d_mask, 4 * words);
            grow(ds.d_off, 4 * words);
            grow(ds.d_key_slot, 4 * ctx->dev_cap);
            grow(ds.d_idx, 4 * (ctx->dev_cap + 2));
            grow(ds.d_scal, 64 * ctx->dev_cap);
            if (grow.rc) return grow.rc;
        }
        {
            cudaMemPoolProps pp; memset(&pp, 0, sizeof pp);
            pp.allocType = cudaMemAllocationTypePinned;
            pp.location.type = cudaMemLocationTypeDevice;
            pp.location.id = dv.id;
            cudaMemPool_t pool = nullptr;
            CK(ctx, cudaMemPoolCreate(&pool, &pp));
            dv.scal_pool.reset(pool);
            uint64_t keep = UINT64_MAX;
            CK(ctx, cudaMemPoolSetAttribute(dv.scal_pool.get(), cudaMemPoolAttrReleaseThreshold, &keep));
            int no = 0;
            CK(ctx, cudaMemPoolSetAttribute(dv.scal_pool.get(), cudaMemPoolReuseAllowInternalDependencies, &no));
        }
        if (!fresh) continue;
#if FAB_G_TWO_LEVEL
        {
            DevArray<u256> d_scratch; DevArray<aff> d_small;
            const size_t nsmall = ((size_t)1 << (FAB_WG / 2)) - 1;
            const size_t threads = (size_t)FAB_G_WINDOWS * 2;
            grow(d_scratch, threads * 2 * nsmall * sizeof(u256));
            grow(d_small, threads * nsmall * sizeof(aff));
            if (grow.rc) return grow.rc;
            small_tables_kernel<<<(unsigned)((threads + 31) / 32), 32, 0, dv.slot[0].stream.get()>>>(nullptr, 1, FAB_WG, FAB_G_WINDOWS, d_small.get(), d_scratch.get(), nullptr);
            const size_t threads2 = (size_t)FAB_G_WINDOWS * ((FAB_G_ENTRIES + FAB_TAB_CHUNK - 1) / FAB_TAB_CHUNK);
            full_tables_kernel<<<(unsigned)((threads2 + 127) / 128), 128, 0, dv.slot[0].stream.get()>>>(d_small.get(), nullptr, nullptr, 1, FAB_WG, FAB_G_WINDOWS, dv.tab->gtab.get());
            ctx->launches += 2;
            CK(ctx, cudaGetLastError());
            CK(ctx, cudaStreamSynchronize(dv.slot[0].stream.get()));
        }
#else
        build_g_table_kernel<<<(unsigned)((tab_entries + 127) / 128), 128, 0, dv.slot[0].stream.get()>>>(dv.tab->gtab.get());
        ctx->launches++;
        CK(ctx, cudaGetLastError());
#endif
    }
    const size_t hwords = (round_up32(max_batch) / 32) + ids.size();
    for (auto& hs : ctx->hslot) {
        Grow grow{ctx};
        for (auto& p : hs.h_in) grow(p, 32 * round_up32(max_batch));
        grow(hs.h_mask, 4 * hwords);
        grow(hs.h_off, 4 * hwords);
        grow(hs.h_key_slot, 4 * round_up32(max_batch));
        if (grow.rc) return grow.rc;
        for (size_t i = 0; i < round_up32(max_batch); i++) hs.h_key_slot.get()[i] = -1;
    }
    for (auto& dv : ctx->devs) {
        CK(ctx, cudaSetDevice(dv.id));
        CK(ctx, cudaStreamSynchronize(dv.slot[0].stream.get()));
    }
    return FABGPU_OK;
}

}  // namespace

extern "C" {

static int create(const int* device_ids, int n_dev, size_t max_batch, const fabgpu_ctx* with, fabgpu_ctx** out)
{
    fabgpu_ctx* ctx = new fabgpu_ctx();
    int rc = init_impl(ctx, device_ids, n_dev, max_batch, with);
    if (rc != FABGPU_OK) {
        g_init_error = ctx->last_error;
        delete ctx;
        return rc;
    }
    *out = ctx;
    return FABGPU_OK;
}

int fabgpu_init(const int* device_ids, int n_dev, size_t max_batch, fabgpu_ctx** out)
{
    if (!out) return FABGPU_E_ARG;
    *out = nullptr;
    return create(device_ids, n_dev, max_batch, nullptr, out);
}

int fabgpu_init_shared(fabgpu_ctx* with, size_t max_batch, fabgpu_ctx** out)
{
    if (!out) return FABGPU_E_ARG;
    *out = nullptr;
    if (!with) { g_init_error = "fabgpu_init_shared needs a context to share tables with"; return FABGPU_E_ARG; }
    return create(nullptr, 0, max_batch, with, out);
}

void fabgpu_destroy(fabgpu_ctx* ctx)
{
    if (!ctx) return;
    for (int s = 0; s < FABGPU_SLOTS; s++) wait_slot(ctx, s);
    delete ctx;
}

const char* fabgpu_last_error(const fabgpu_ctx* ctx) { return ctx ? ctx->last_error.c_str() : g_init_error.c_str(); }
int fabgpu_device_count(const fabgpu_ctx* ctx) { return ctx ? (int)ctx->devs.size() : 0; }
size_t fabgpu_max_batch(const fabgpu_ctx* ctx) { return ctx ? ctx->max_batch : 0; }
unsigned long long fabgpu_launch_count(const fabgpu_ctx* ctx) { return ctx ? ctx->launches.load() : 0ull; }

int fabgpu_host_buffers(fabgpu_ctx* ctx, int slot, uint8_t** qx, uint8_t** qy, uint8_t** e, uint8_t** r, uint8_t** s,
                        uint32_t** mask, uint32_t** offcurve)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    HostSlot& hs = ctx->hslot[slot];
    if (qx) *qx = hs.h_in[0].get();
    if (qy) *qy = hs.h_in[1].get();
    if (e) *e = hs.h_in[2].get();
    if (r) *r = hs.h_in[3].get();
    if (s) *s = hs.h_in[4].get();
    if (mask) *mask = hs.h_mask.get();
    if (offcurve) *offcurve = hs.h_off.get();
    return FABGPU_OK;
}

static int verify_async_impl(fabgpu_ctx* ctx, int slot, size_t n, bool keyed)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);     // handles -> slots -> enqueue, see KeyTables
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n > ctx->max_batch) { ctx->last_error = "n exceeds max_batch"; return FABGPU_E_ARG; }
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    return enqueue_slot(ctx, slot, n, keyed);
}

int fabgpu_verify_p256_async(fabgpu_ctx* ctx, int slot, size_t n) { return verify_async_impl(ctx, slot, n, false); }
int fabgpu_verify_p256_keyed_async(fabgpu_ctx* ctx, int slot, size_t n) { return verify_async_impl(ctx, slot, n, true); }

int fabgpu_verify_p256_keyed(fabgpu_ctx* ctx, int slot, size_t n)
{
    int rc = fabgpu_verify_p256_keyed_async(ctx, slot, n);
    if (rc) return rc;
    return fabgpu_wait(ctx, slot);
}

int fabgpu_host_key_slots(fabgpu_ctx* ctx, int slot, int32_t** key_slot)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || !key_slot) return FABGPU_E_ARG;
    *key_slot = ctx->hslot[slot].h_key_slot.get();
    return FABGPU_OK;
}

int fabgpu_key_slot_capacity(const fabgpu_ctx* ctx) { return ctx ? ctx->kt->key_slots : 0; }

// Looks the keys up in the table cache and builds tables for the missing ones (one launch per device for the whole set).
int fabgpu_keys_register(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, int32_t* slots_out)
{
    if (!ctx || K < 0 || (K && (!keys_xy || !slots_out))) return FABGPU_E_ARG;
    // Fast path under the shared lock: every key already owns a table (the steady state of KeyImport / resolve_key_tables).
    {
        std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);
        std::lock_guard<std::mutex> lk(ctx->kt->mu);
        bool all = true;
        for (int k = 0; k < K && all; k++) all = ctx->kt->key_map.count(std::string((const char*)keys_xy + 64 * (size_t)k, 64)) != 0;
        if (all) {
            ctx->kt->tick++;
            for (int k = 0; k < K; k++) {
                const int sl = ctx->kt->key_map[std::string((const char*)keys_xy + 64 * (size_t)k, 64)];
                slots_out[k] = make_handle(ctx, sl); ctx->kt->slot_tick[sl] = ctx->kt->tick;
            }
            return FABGPU_OK;
        }
    }
    std::unique_lock<std::shared_mutex> wl(ctx->kt->tab_mu);
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::lock_guard<std::mutex> kl(ctx->kt->mu);
    std::vector<int> fresh;                      // indices into keys_xy that need a table
    std::vector<int32_t> fresh_slot;
    std::vector<char> slot_taken(ctx->kt->key_slots, 0);
    ctx->kt->tick++;
    for (int k = 0; k < K; k++) {
        std::string key((const char*)keys_xy + 64 * (size_t)k, 64);
        auto it = ctx->kt->key_map.find(key);
        if (it != ctx->kt->key_map.end()) { slots_out[k] = make_handle(ctx, it->second); ctx->kt->slot_tick[it->second] = ctx->kt->tick; slot_taken[it->second] = 1; continue; }
        // least recently used slot that this call has not touched
        int best = -1;
        for (int sl = 0; sl < ctx->kt->key_slots; sl++)
            if (!slot_taken[sl] && (best < 0 || ctx->kt->slot_tick[sl] < ctx->kt->slot_tick[best])) best = sl;
        if (best < 0) { slots_out[k] = -1; continue; }            // more distinct keys in one call than slots: stays generic
        // The slot's old owner loses it NOW (its handles die with the generation bump), but the new key is mapped only after
        // its table exists on every device: a failure below leaves the slot empty, never pointing at another key's table.
        if (!ctx->kt->slot_key[best].empty()) { ctx->kt->key_map.erase(ctx->kt->slot_key[best]); ctx->kt->slot_key[best].clear(); ctx->kt->slot_gen[best]++; }
        ctx->kt->slot_tick[best] = ctx->kt->tick; slot_taken[best] = 1;
        slots_out[k] = -1;
        fresh.push_back(k); fresh_slot.push_back(best);
    }
    if (fresh.empty()) return FABGPU_OK;
    const int F = (int)fresh.size();
    std::vector<uint8_t> fk(64 * (size_t)F);
    for (int i = 0; i < F; i++) memcpy(fk.data() + 64 * (size_t)i, keys_xy + 64 * (size_t)fresh[i], 64);
    std::vector<uint32_t> flags(F, 0);
    auto build_on = [&](Device& dv) -> int {
        CK(ctx, cudaSetDevice(dv.id));
        // an evicted slot's table may still be read by a batch in flight: drain this device first (registration is rare)
        for (auto& ds : dv.slot) CK(ctx, cudaStreamSynchronize(ds.stream.get()));
        CK(ctx, cudaDeviceSynchronize());            // launches on caller streams (fabgpu_verify_p256_device_keyed) as well
        DevArray<uint8_t> d_keys; DevArray<int32_t> d_slots; DevArray<uint32_t> d_flags; DevArray<u256> d_scratch;
        Grow grow{ctx};
        grow(d_keys, fk.size());
        grow(d_slots, 4 * (size_t)F);
        grow(d_flags, 4 * (size_t)F);
        if (grow.rc) return grow.rc;
        CK(ctx, cudaMemcpy(d_keys.get(), fk.data(), fk.size(), cudaMemcpyHostToDevice));
        CK(ctx, cudaMemcpy(d_slots.get(), fresh_slot.data(), 4 * (size_t)F, cudaMemcpyHostToDevice));
#if FAB_Q_TWO_LEVEL
        DevArray<aff> d_small;
        const size_t nsmall = ((size_t)1 << (FAB_WQ / 2)) - 1;
        const size_t threads = (size_t)F * FAB_Q_WINDOWS * 2;
        grow(d_scratch, threads * 2 * nsmall * sizeof(u256));
        grow(d_small, threads * nsmall * sizeof(aff));
        if (grow.rc) return grow.rc;
        small_tables_kernel<<<(unsigned)((threads + 31) / 32), 32, 0, dv.slot[0].stream.get()>>>(d_keys.get(), F, FAB_WQ, FAB_Q_WINDOWS, d_small.get(), d_scratch.get(), d_flags.get());
        const size_t threads2 = (size_t)F * FAB_Q_WINDOWS * ((FAB_Q_ENTRIES + FAB_TAB_CHUNK - 1) / FAB_TAB_CHUNK);
        full_tables_kernel<<<(unsigned)((threads2 + 127) / 128), 128, 0, dv.slot[0].stream.get()>>>(d_small.get(), d_slots.get(), d_flags.get(), F, FAB_WQ, FAB_Q_WINDOWS, dv.tab->qtab.get());
        ctx->launches += 2;
#else
        const size_t threads = (size_t)F * FAB_Q_WINDOWS;
        grow(d_scratch, threads * 2 * FAB_Q_ENTRIES * sizeof(u256));
        if (grow.rc) return grow.rc;
        build_key_tables_kernel<<<(unsigned)((threads + 31) / 32), 32, 0, dv.slot[0].stream.get()>>>(d_keys.get(), d_slots.get(), F, dv.tab->qtab.get(), d_scratch.get(), d_flags.get());
        ctx->launches++;
#endif
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaStreamSynchronize(dv.slot[0].stream.get()));
        CK(ctx, cudaMemcpy(flags.data(), d_flags.get(), 4 * (size_t)F, cudaMemcpyDeviceToHost));
        return FABGPU_OK;
    };
    for (auto& dv : ctx->devs) {
        const int rc = build_on(dv);
        if (rc) return rc;                        // nothing was committed: the recycled slots stay empty (handles -1), the keys stay generic
    }
    for (int i = 0; i < F; i++) {
        if (!flags[i]) continue;                  // not a curve point: no table; the generic kernel reports it as off-curve
        const int sl = fresh_slot[i];
        std::string key((const char*)fk.data() + 64 * (size_t)i, 64);
        ctx->kt->slot_key[sl] = key; ctx->kt->key_map[key] = sl;
        slots_out[fresh[i]] = make_handle(ctx, sl);
    }
    return FABGPU_OK;
}

// Small tables for the keys that have none yet; handles_out[k] = small handle, or -1 when no slot could be had.  The builds are
// enqueued on every device's build stream and NOT waited for: consumers order themselves behind Device::s_ev (launch_verify).
// Caller holds neither tab_mu nor mu.
static int small_register(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, int32_t* handles_out)
{
    if (ctx->kt->small_slots <= 0) { for (int k = 0; k < K; k++) handles_out[k] = -1; return FABGPU_OK; }
    {   // fast path under the shared lock: every key already owns a small table
        std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);
        std::lock_guard<std::mutex> lk(ctx->kt->mu);
        bool all = true;
        KeyTables::Key64 kk;
        for (int k = 0; k < K && all; k++) { memcpy(kk.b, keys_xy + 64 * (size_t)k, 64); all = ctx->kt->small_map.count(kk) != 0; }
        if (all) {
            ctx->kt->tick++;
            for (int k = 0; k < K; k++) {
                memcpy(kk.b, keys_xy + 64 * (size_t)k, 64);
                const int sl = ctx->kt->small_map[kk];
                handles_out[k] = make_small_handle(ctx, sl); ctx->kt->small_tick[sl] = ctx->kt->tick;
            }
            return FABGPU_OK;
        }
    }
    const bool trace = getenv("FABGPU_TRACE") != nullptr;
    auto tnow = [] { return std::chrono::steady_clock::now(); };
    auto tus = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
    auto tr0 = tnow();
    std::unique_lock<std::shared_mutex> wl(ctx->kt->tab_mu);
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::lock_guard<std::mutex> kl(ctx->kt->mu);
    auto tr1 = tnow();
    ctx->kt->tick++;
    std::vector<int> fresh; std::vector<int32_t> fresh_slot;
    KeyTables::Key64 kk;
    int need = 0;
    for (int k = 0; k < K; k++) { memcpy(kk.b, keys_xy + 64 * (size_t)k, 64); if (!ctx->kt->small_map.count(kk)) need++; }
    if (need > (int)ctx->kt->small_free.size()) {
        // Out of free slots: recycle the least recently used ones in bulk (an eighth of the pool at least), after draining every device --
        // a batch in flight may still read them.  Rare by construction: the pool holds thousands of keys.
        for (auto& dv : ctx->devs) { CK(ctx, cudaSetDevice(dv.id)); CK(ctx, cudaDeviceSynchronize()); }
        std::vector<int> order;
        for (int sl = 0; sl < ctx->kt->small_slots; sl++) if (ctx->kt->small_used[sl]) order.push_back(sl);
        // keys of THIS call keep their tables
        for (int k = 0; k < K; k++) { memcpy(kk.b, keys_xy + 64 * (size_t)k, 64); auto it = ctx->kt->small_map.find(kk); if (it != ctx->kt->small_map.end()) ctx->kt->small_tick[it->second] = ctx->kt->tick; }
        std::sort(order.begin(), order.end(), [&](int a, int b) { return ctx->kt->small_tick[a] < ctx->kt->small_tick[b]; });
        const size_t want = std::max<size_t>((size_t)need - ctx->kt->small_free.size(), (size_t)ctx->kt->small_slots / 8);
        for (size_t i = 0; i < order.size() && i < want; i++) {
            const int sl = order[i];
            if (ctx->kt->small_tick[sl] == ctx->kt->tick) break;
            ctx->kt->small_map.erase(ctx->kt->small_key[sl]); ctx->kt->small_used[sl] = 0; ctx->kt->small_gen[sl]++;
            ctx->kt->small_free.push_back(sl); ctx->kt->small_recycled++;
        }
    }
    for (int k = 0; k < K; k++) {
        memcpy(kk.b, keys_xy + 64 * (size_t)k, 64);
        auto it = ctx->kt->small_map.find(kk);
        if (it != ctx->kt->small_map.end()) { handles_out[k] = make_small_handle(ctx, it->second); ctx->kt->small_tick[it->second] = ctx->kt->tick; continue; }
        handles_out[k] = -1;
        if (ctx->kt->small_free.empty()) continue;                      // more distinct keys in one call than the pool holds: stays generic
        const int sl = ctx->kt->small_free.back(); ctx->kt->small_free.pop_back();
        // mapped at once (a duplicate later in this call finds it); un-mapped again below if the enqueue fails
        ctx->kt->small_map[kk] = sl; ctx->kt->small_key[sl] = kk; ctx->kt->small_used[sl] = 1; ctx->kt->small_tick[sl] = ctx->kt->tick;
        fresh.push_back(k); fresh_slot.push_back(sl);
        handles_out[k] = make_small_handle(ctx, sl);
    }
    if (fresh.empty()) return FABGPU_OK;
    const int F = (int)fresh.size();
    ctx->kt->small_built += (unsigned long long)F;
    std::vector<uint8_t> fk(64 * (size_t)F);
    for (int i = 0; i < F; i++) memcpy(fk.data() + 64 * (size_t)i, keys_xy + 64 * (size_t)fresh[i], 64);
    auto tr2 = tnow();
    auto build_on = [&](Device& dv) -> int {
        CK(ctx, cudaSetDevice(dv.id));
        auto b0 = tnow();
        if ((size_t)F > dv.tab->s_cap()) {
            CK(ctx, cudaStreamSynchronize(dv.tab->s_stream.get()));            // an earlier build may still use the scratch
            const size_t c = (size_t)F + (size_t)F / 2 + 256;
            Grow grow{ctx};
            grow(dv.tab->s_keys, 64 * c);
            grow(dv.tab->s_slots, 4 * c);
            grow(dv.tab->s_bases, c * FAB_S_WINDOWS * sizeof(aff));      // last: it holds s_cap()
            if (grow.rc) return grow.rc;
        }
        auto b1 = tnow();
        CK(ctx, cudaMemcpyAsync(dv.tab->s_keys.get(), fk.data(), fk.size(), cudaMemcpyHostToDevice, dv.tab->s_stream.get()));
        CK(ctx, cudaMemcpyAsync(dv.tab->s_slots.get(), fresh_slot.data(), 4 * (size_t)F, cudaMemcpyHostToDevice, dv.tab->s_stream.get()));
        CK(ctx, cudaStreamSynchronize(dv.tab->s_stream.get()));                // the sources are local vectors
        auto b2 = tnow();
        small_bases_kernel<<<(unsigned)((F + 31) / 32), 32, 0, dv.tab->s_stream.get()>>>(dv.tab->s_keys.get(), dv.tab->s_slots.get(), F, dv.tab->s_bases.get(), dv.tab->stab.get());
        small_windows_kernel<<<(unsigned)(((size_t)F * FAB_S_WINDOWS + 127) / 128), 128, 0, dv.tab->s_stream.get()>>>(dv.tab->s_bases.get(), dv.tab->s_slots.get(), F, dv.tab->stab.get());
        ctx->launches += 2;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaEventRecord(dv.tab->s_ev.get(), dv.tab->s_stream.get()));
        dv.tab->s_ev_set = true;
        if (trace) fprintf(stderr, "[fabgpu] small_register F=%d: lock %.0f us, bookkeeping %.0f us, scratch %.0f us, copies %.0f us, launches %.0f us\n", F, tus(tr0, tr1),
                           tus(tr1, tr2), tus(b0, b1), tus(b1, b2), tus(b2, tnow()));
        return FABGPU_OK;
    };
    for (auto& dv : ctx->devs) {
        const int rc = build_on(dv);
        if (rc) {                                                   // nothing usable was built: give the slots back, the keys stay generic
            for (int i = 0; i < F; i++) {
                const int sl = fresh_slot[i];
                ctx->kt->small_map.erase(ctx->kt->small_key[sl]); ctx->kt->small_used[sl] = 0; ctx->kt->small_gen[sl]++; ctx->kt->small_free.push_back(sl);
                handles_out[fresh[i]] = -1;
            }
            return rc;
        }
    }
    return FABGPU_OK;
}

int fabgpu_keys_register_small(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, int32_t* handles_out)
{
    if (!ctx || K < 0 || (K && (!keys_xy || !handles_out))) return FABGPU_E_ARG;
    return small_register(ctx, keys_xy, K, handles_out);
}
int fabgpu_small_slot_capacity(const fabgpu_ctx* ctx) { return ctx ? ctx->kt->small_slots : 0; }
void fabgpu_small_table_info(int* window_bits, int* windows, size_t* table_bytes)
{
    if (window_bits) *window_bits = FAB_WS;
    if (windows) *windows = FAB_S_WINDOWS;
    if (table_bytes) *table_bytes = (size_t)FAB_S_POINTS * sizeof(aff);
}
int fabgpu_key_table_stats(fabgpu_ctx* ctx, unsigned long long out[4])
{
    if (!ctx || !out) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->kt->mu);
    out[0] = ctx->kt->key_map.size(); out[1] = ctx->kt->small_map.size(); out[2] = ctx->kt->small_built; out[3] = ctx->kt->small_recycled;
    return FABGPU_OK;
}

int fabgpu_wait(fabgpu_ctx* ctx, int slot)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    // No context lock: waiting on one slot's streams must not block the enqueue of another slot (the provider's aggregator
    // fills slot k+1 while slot k runs).  Stream handles are immutable after fabgpu_init; errors go to a local string first.
    for (auto& dv : ctx->devs) {
        cudaError_t e = cudaSetDevice(dv.id);
        if (e == cudaSuccess) e = cudaStreamSynchronize(dv.slot[slot].stream.get());
        if (e != cudaSuccess) {
            std::lock_guard<std::mutex> lk(ctx->mu);
            ctx->last_error = std::string("cudaStreamSynchronize failed: ") + cudaGetErrorString(e);
            return FABGPU_E_CUDA;
        }
    }
    return FABGPU_OK;
}

int fabgpu_verify_p256(fabgpu_ctx* ctx, int slot, size_t n)
{
    int rc = fabgpu_verify_p256_async(ctx, slot, n);
    if (rc) return rc;
    return fabgpu_wait(ctx, slot);
}

int fabgpu_verify_p256_host(fabgpu_ctx* ctx, const uint8_t* qx, const uint8_t* qy, const uint8_t* e, const uint8_t* r,
                            const uint8_t* s, size_t n, uint32_t* mask, uint32_t* offcurve)
{
    if (!ctx || (n && (!qx || !qy || !e || !r || !s || !mask))) return FABGPU_E_ARG;
    if (n > ctx->max_batch) { ctx->last_error = "n exceeds max_batch"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    HostSlot& hs = ctx->hslot[0];
    const uint8_t* src[5] = {qx, qy, e, r, s};
    for (int a = 0; a < 5; a++) memcpy(hs.h_in[a].get(), src[a], 32 * n);
    int rc = fabgpu_verify_p256(ctx, 0, n);
    if (rc) return rc;
    const size_t words = (n + 31) / 32;
    memcpy(mask, hs.h_mask.get(), 4 * words);
    if (offcurve) memcpy(offcurve, hs.h_off.get(), 4 * words);
    return FABGPU_OK;
}

int fabgpu_verify_p256_device(fabgpu_ctx* ctx, int dev_index, const void* d_qx, const void* d_qy, const void* d_e,
                              const void* d_r, const void* d_s, size_t n, void* d_mask, void* d_offcurve, void* cuda_stream)
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size()) return FABGPU_E_ARG;
    if (n && (!d_qx || !d_qy || !d_e || !d_r || !d_s || !d_mask)) return FABGPU_E_ARG;
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    Device& dv = ctx->devs[dev_index];
    CK(ctx, cudaSetDevice(dv.id));
    cudaStream_t st = (cudaStream_t)cuda_stream;   // NULL is CUDA's default stream, exactly as in the runtime API
    return launch_verify(ctx, dv, MODE_GENERIC, nullptr, (const uint8_t*)d_qx, (const uint8_t*)d_qy, (const uint8_t*)d_e,
                         (const uint8_t*)d_r, (const uint8_t*)d_s, n, (uint32_t*)d_mask, (uint32_t*)d_offcurve, st);
}

int fabgpu_verify_p256_device_keyed(fabgpu_ctx* ctx, int dev_index, int all_cached, const void* d_key_slot, const void* d_qx,
                                    const void* d_qy, const void* d_e, const void* d_r, const void* d_s, size_t n, void* d_mask,
                                    void* d_offcurve, void* cuda_stream)
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size()) return FABGPU_E_ARG;
    if (n && (!d_key_slot || !d_e || !d_r || !d_s || !d_mask)) return FABGPU_E_ARG;
    if (n && !all_cached && (!d_qx || !d_qy)) return FABGPU_E_ARG;
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    Device& dv = ctx->devs[dev_index];
    CK(ctx, cudaSetDevice(dv.id));
    return launch_verify(ctx, dv, all_cached == 2 ? MODE_SMALL : (all_cached ? MODE_CACHED : MODE_MIXED), (const int32_t*)d_key_slot, (const uint8_t*)d_qx,
                         (const uint8_t*)d_qy, (const uint8_t*)d_e, (const uint8_t*)d_r, (const uint8_t*)d_s, n, (uint32_t*)d_mask,
                         (uint32_t*)d_offcurve, (cudaStream_t)cuda_stream);
}

// ---- bitmask exchange over peer memory -------------------------------------------------------------------------------------
static const int kPeerGens = 2;
static size_t peer_buf_words(int world, size_t wpr) { return (size_t)kPeerGens * world * wpr + FAB_PEER_MAX; }

int fabgpu_peer_mask_create(fabgpu_ctx* ctx, int dev_index, int world, int rank, size_t words_per_rank, uint8_t handle_out[FABGPU_IPC_HANDLE_BYTES])
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size() || world < 1 || world > FAB_PEER_MAX || rank < 0 || rank >= world || !words_per_rank || !handle_out)
        return FABGPU_E_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) <= FABGPU_IPC_HANDLE_BYTES, "IPC handle size");
    Device& dv = ctx->devs[dev_index];
    auto& pr = dv.peer;
    if (pr.local.get()) { ctx->last_error = "peer mask already created on this device"; return FABGPU_E_ARG; }
    CK(ctx, cudaSetDevice(dv.id));
    const size_t bytes = 4 * peer_buf_words(world, words_per_rank);
    if (int rc = pr.local.reserve(ctx, bytes)) return rc;
    CK(ctx, cudaMemset(pr.local.get(), 0, bytes));
    if (int rc = pr.done.reserve(ctx, 8)) return rc;
    CK(ctx, cudaMemset(pr.done.get(), 0, 8));
    pr.timeout = pr.done.get() + 1;
    if (int rc = pr.h_timeout.reserve(ctx, 4)) return rc;
    *pr.h_timeout.get() = 0;
    cudaIpcMemHandle_t h;
    CK(ctx, cudaIpcGetMemHandle(&h, pr.local.get()));
    memset(handle_out, 0, FABGPU_IPC_HANDLE_BYTES);
    memcpy(handle_out, &h, sizeof h);
    pr.world = world; pr.rank = rank; pr.words_per_rank = words_per_rank;
    pr.ready = world == 1;
    return FABGPU_OK;
}

int fabgpu_peer_mask_open(fabgpu_ctx* ctx, int dev_index, const uint8_t* handles)
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size() || !handles) return FABGPU_E_ARG;
    Device& dv = ctx->devs[dev_index];
    auto& pr = dv.peer;
    if (!pr.local.get()) { ctx->last_error = "fabgpu_peer_mask_create first"; return FABGPU_E_ARG; }
    CK(ctx, cudaSetDevice(dv.id));
    for (int p = 0; p < pr.world; p++) {
        if (p == pr.rank || pr.mapped[p]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + (size_t)p * FABGPU_IPC_HANDLE_BYTES, sizeof h);
        void* m = nullptr;
        CK(ctx, cudaIpcOpenMemHandle(&m, h, cudaIpcMemLazyEnablePeerAccess));
        pr.mapped[p].reset((uint32_t*)m);
    }
    pr.ready = true;
    return FABGPU_OK;
}

int fabgpu_peer_mask_close(fabgpu_ctx* ctx, int dev_index)
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size()) return FABGPU_E_ARG;
    Device& dv = ctx->devs[dev_index];
    auto& pr = dv.peer;
    cudaSetDevice(dv.id);
    cudaDeviceSynchronize();
    std::exchange(pr, Device::Peer());      // the old state goes at the end of the statement: mappings closed first (Device::Peer)
    return FABGPU_OK;
}

int fabgpu_verify_p256_device_keyed_allgather(fabgpu_ctx* ctx, int dev_index, int all_cached, const void* d_key_slot, const void* d_qx,
                                              const void* d_qy, const void* d_e, const void* d_r, const void* d_s, size_t n, uint32_t step,
                                              void** d_full_mask, void* cuda_stream)
{
    if (!ctx || dev_index < 0 || dev_index >= (int)ctx->devs.size() || !d_full_mask || step == 0) return FABGPU_E_ARG;
    if (n && (!d_key_slot || !d_e || !d_r || !d_s)) return FABGPU_E_ARG;
    if (n && !all_cached && (!d_qx || !d_qy)) return FABGPU_E_ARG;
    Device& dv = ctx->devs[dev_index];
    auto& pr = dv.peer;
    if (!pr.ready) { ctx->last_error = "peer masks are not set up (fabgpu_peer_mask_create / _open)"; return FABGPU_E_ARG; }
    if ((n + 31) / 32 > pr.words_per_rank) { ctx->last_error = "batch exceeds words_per_rank"; return FABGPU_E_ARG; }
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    if (*pr.h_timeout.get()) { ctx->last_error = "a peer did not publish its bitmask in time"; return FABGPU_E_CUDA; }
    CK(ctx, cudaSetDevice(dv.id));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    PeerOut po; memset(&po, 0, sizeof po);
    for (int p = 0; p < pr.world; p++) po.buf[p] = pr.buf(p);
    po.done = pr.done.get(); po.world = (uint32_t)pr.world; po.rank = (uint32_t)pr.rank; po.words_per_rank = (uint32_t)pr.words_per_rank;
    po.gen_off = (uint32_t)((step % kPeerGens) * pr.world * pr.words_per_rank);
    po.flag_off = (uint32_t)((size_t)kPeerGens * pr.world * pr.words_per_rank);
    po.step = step;
    // the rank's own words also land in its local segment (buf[rank] is the local buffer): `mask` for the kernels is that segment
    uint32_t* local_seg = pr.local.get() + po.gen_off + (size_t)pr.rank * pr.words_per_rank;
    int rc = launch_verify(ctx, dv, all_cached == 2 ? MODE_SMALL : (all_cached ? MODE_CACHED : MODE_MIXED), (const int32_t*)d_key_slot, (const uint8_t*)d_qx, (const uint8_t*)d_qy,
                           (const uint8_t*)d_e, (const uint8_t*)d_r, (const uint8_t*)d_s, n, local_seg, nullptr, st, nullptr, 0, &po);
    if (rc) return rc;
    peer_wait_kernel<<<1, 32, 0, st>>>(pr.local.get() + po.flag_off, po.world, step, pr.timeout);
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(pr.h_timeout.get(), pr.timeout, 4, cudaMemcpyDeviceToHost, st));
    *d_full_mask = pr.local.get() + po.gen_off;
    return FABGPU_OK;
}

int fabgpu_gate_signature(const uint8_t* sig, size_t sig_len, uint8_t r_out[32], uint8_t s_out[32])
{
    host::Gate g;
    host::gate_signature(sig, sig_len, g, false);
    if (g.status == FABGPU_ST_VALID) { memcpy(r_out, g.r, 32); memcpy(s_out, g.s, 32); }
    return g.status;
}


// fabgpu_bccsp_verify_batch with the gates on the device: the host only stages the raw blobs into pinned memory
// (parallel streaming copies) and reads one status byte per signature back.  Device 0 of the context.
// Device-gated batch, first half: stage into the slot's pinned buffers and enqueue copies + three kernels + the status
// read-back on the slot's stream.  Returns without waiting; the caller's buffers are no longer referenced.
// Grows the slot's pinned + device buffers of the device-gated batch path to the given capacities.
static int gate_bufs_reserve(fabgpu_ctx* ctx, int slot, size_t n, size_t sig_bytes, size_t dig_bytes, size_t K)
{
    auto& gb = ctx->gb[slot];
    Grow grow{ctx};
    if (n > gb.n_cap()) {
        const size_t c = round_up32(n + (n >> 2) + 1024);
        grow(gb.h_sig_off, 4 * (c + 1)); grow(gb.h_dig_off, 4 * (c + 1)); grow(gb.h_kidx, 4 * c); grow(gb.h_status, c);
        grow(gb.d_sig_off, 4 * (c + 1)); grow(gb.d_dig_off, 4 * (c + 1)); grow(gb.d_kidx, 4 * c);
        grow(gb.d_status, c); grow(gb.d_pre, c); grow(gb.d_r, 32 * c); grow(gb.d_s, 32 * c);
        grow(gb.d_e, 32 * c); grow(gb.d_qx, 32 * c); grow(gb.d_qy, 32 * c); grow(gb.d_ks, 4 * c);
        grow(gb.d_mask, c / 8 + 8); grow(gb.d_off, c / 8 + 8); grow(gb.d_idx, 4 * (c + 2));
        grow(gb.d_scal, 64 * c);
        if (grow.rc) return grow.rc;
    }
    if (sig_bytes > gb.sig_cap()) { const size_t c = sig_bytes + (sig_bytes >> 2) + 4096; grow(gb.h_sigs, c); grow(gb.d_sigs, c); if (grow.rc) return grow.rc; }
    if (dig_bytes > gb.dig_cap()) { const size_t c = dig_bytes + (dig_bytes >> 2) + 4096; grow(gb.h_digs, c); grow(gb.d_digs, c); if (grow.rc) return grow.rc; }
    if (K > gb.k_cap()) { const size_t c = K + 64; grow(gb.h_keys, 64 * c); grow(gb.h_slot_of, 4 * c); grow(gb.d_keys, 64 * c); grow(gb.d_slot_of, 4 * c); }
    return grow.rc;
}

// inplace: the batch already lies in the slot's pinned buffers (fabgpu_bccsp_batch_buffers): nothing is staged.
static int bccsp_device_submit(fabgpu_ctx* ctx, int slot, const uint8_t* keys_xy, int K, const int32_t* key_idx, const uint8_t* digests,
                               const uint32_t* dig_off, const uint8_t* sigs, const uint32_t* sig_off, size_t n,
                               const std::vector<int32_t>& slot_of, bool inplace = false)
{
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::micro>(b - a).count();
    };
    auto t0 = now();
    Device& dv = ctx->devs[0];
    DevSlot& ds = dv.slot[slot];
    auto& gb = ctx->gb[slot];
    CK(ctx, cudaSetDevice(dv.id));
    // sig_off / dig_off may be a window of a longer table (a chunk of a call): bytes [off[0], off[n]) of the blobs belong to it
    const uint32_t sig_base = sig_off[0], dig_base = dig_off[0];
    const size_t sig_bytes = sig_off[n] - sig_base, dig_bytes = dig_off[n] - dig_base;
    int rc = gate_bufs_reserve(ctx, slot, n, sig_bytes, dig_bytes, (size_t)(K > 0 ? K : 0));
    if (rc) return rc;
    // stage: every host thread copies its slice of each array
    const int T = ctx->pool->size();
    bool all_slots = K > 0;
    int classes = K > 0 ? 0 : CLASS_GENERIC;                  // which non-big classes the batch holds (signatures with a bad key index are decided by the gates)
    std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);      // held until the verify kernel is enqueued: the slots cannot be recycled in between
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (int k = 0; k < K; k++) {
            gb.h_slot_of.get()[k] = handle_to_slot(ctx, slot_of[k]);
            if (gb.h_slot_of.get()[k] < 0) all_slots = false;
            if (gb.h_slot_of.get()[k] == -1) classes |= CLASS_GENERIC; else if (gb.h_slot_of.get()[k] <= -2) classes |= CLASS_SMALL;
        }
    }
    if (K > 0 && !inplace) memcpy(gb.h_keys.get(), keys_xy, 64 * (size_t)K);
    if (!inplace) ctx->pool->run([&](int tid) {
        auto slice = [&](size_t total, size_t& lo, size_t& hi) { lo = total * (size_t)tid / T; hi = total * (size_t)(tid + 1) / T; };
        size_t lo, hi;
        slice(sig_bytes, lo, hi); stage_copy(gb.h_sigs.get() + lo, sigs + sig_base + lo, hi - lo);
        slice(dig_bytes, lo, hi); stage_copy(gb.h_digs.get() + lo, digests + dig_base + lo, hi - lo);
        slice(4 * (n + 1), lo, hi); stage_copy((uint8_t*)gb.h_sig_off.get() + lo, (const uint8_t*)sig_off + lo, hi - lo);
        slice(4 * (n + 1), lo, hi); stage_copy((uint8_t*)gb.h_dig_off.get() + lo, (const uint8_t*)dig_off + lo, hi - lo);
        slice(4 * n, lo, hi); stage_copy((uint8_t*)gb.h_kidx.get() + lo, (const uint8_t*)key_idx + lo, hi - lo);
        stage_fence();
    });
    auto t1 = now();
    cudaStream_t st = ds.stream.get();
    CK(ctx, cudaMemcpyAsync(gb.d_sigs.get(), gb.h_sigs.get(), sig_bytes, cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(gb.d_digs.get(), gb.h_digs.get(), dig_bytes, cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(gb.d_sig_off.get(), gb.h_sig_off.get(), 4 * (n + 1), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(gb.d_dig_off.get(), gb.h_dig_off.get(), 4 * (n + 1), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(gb.d_kidx.get(), gb.h_kidx.get(), 4 * n, cudaMemcpyHostToDevice, st));
    if (K > 0) {
        CK(ctx, cudaMemcpyAsync(gb.d_keys.get(), gb.h_keys.get(), 64 * (size_t)K, cudaMemcpyHostToDevice, st));
        CK(ctx, cudaMemcpyAsync(gb.d_slot_of.get(), gb.h_slot_of.get(), 4 * (size_t)K, cudaMemcpyHostToDevice, st));
    }
    bdev::bccsp_gate_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(gb.d_sigs.get(), gb.d_sig_off.get(), gb.d_digs.get(), gb.d_dig_off.get(), gb.d_kidx.get(), gb.d_slot_of.get(), gb.d_keys.get(), K,
                                                                        (uint32_t)n, gb.d_r.get(), gb.d_s.get(), gb.d_e.get(), gb.d_ks.get(), (classes & CLASS_GENERIC) ? gb.d_qx.get() : nullptr,
                                                                        (classes & CLASS_GENERIC) ? gb.d_qy.get() : nullptr, gb.d_pre.get(), sig_base, dig_base);
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    rc = launch_verify(ctx, dv, all_slots ? MODE_CACHED : MODE_MIXED, gb.d_ks.get(), gb.d_qx.get(), gb.d_qy.get(), gb.d_e.get(), gb.d_r.get(), gb.d_s.get(), n, gb.d_mask.get(), gb.d_off.get(), st, nullptr, 0, nullptr,
                       gb.d_idx.get(), classes ? classes : CLASS_GENERIC, gb.d_scal.get());
    if (rc) return rc;
    bdev::bccsp_status_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(gb.d_pre.get(), gb.d_mask.get(), gb.d_off.get(), (uint32_t)n, gb.d_status.get());
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(gb.h_status.get(), gb.d_status.get(), n, cudaMemcpyDeviceToHost, st));
    gb.t_submit = t1; gb.n = n;
    ctx->timing[1] = us(t0, t1);
    return FABGPU_OK;
}

// Second half: wait for the slot's stream and hand the statuses out.
static int bccsp_device_finish(fabgpu_ctx* ctx, int slot, uint8_t* status)
{
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::micro>(b - a).count();
    };
    auto& gb = ctx->gb[slot];
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    CK(ctx, cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get()));
    auto t2 = now();
    memcpy(status, gb.h_status.get(), gb.n);
    ctx->timing[2] = us(gb.t_submit, t2); ctx->timing[3] = us(t2, now());
    return FABGPU_OK;
}

// Which table serves each key of a call.  slot_of[k]: handle of key k's big table (>= 0), of its small table (<= -2), or -1.
//   * a key that already owns a table keeps using it, however few signatures it has in this call;
//   * >= key_min_uses signatures in this call earn the big table (what KeyImport does once per identity in the Go provider);
//   * otherwise the key's signatures are counted across calls, and small_min_uses of them earn a small table.
static int resolve_key_tables(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, const int32_t* key_idx, size_t n, std::vector<int32_t>& slot_of)
{
    slot_of.assign(K > 0 ? K : 0, -1);
    if (!(K > 0 && keys_xy && ctx->kt->key_min_uses >= 0)) return FABGPU_OK;
    std::vector<uint32_t> uses(K, 0);
    for (size_t i = 0; i < n; i++) if (key_idx[i] >= 0 && key_idx[i] < K) uses[key_idx[i]]++;
    std::vector<int> want_big, want_small;
    {
        std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);
        std::lock_guard<std::mutex> lk(ctx->kt->mu);
        KeyTables::Key64 kk;
        bool touched = false;
        static thread_local std::string kbuf(64, '\0');          // lookup key without a heap allocation per key
        for (int k = 0; k < K; k++) {
            if (!uses[k]) continue;
            if (!ctx->kt->key_map.empty() || uses[k] >= (uint32_t)ctx->kt->key_min_uses) {
                memcpy(&kbuf[0], keys_xy + 64 * (size_t)k, 64);
                auto it = ctx->kt->key_map.find(kbuf);
                if (it != ctx->kt->key_map.end()) {
                    if (!touched) { ctx->kt->tick++; touched = true; }
                    slot_of[k] = make_handle(ctx, it->second); ctx->kt->slot_tick[it->second] = ctx->kt->tick; continue;
                }
            }
            if (uses[k] >= (uint32_t)ctx->kt->key_min_uses) { want_big.push_back(k); continue; }
            if (ctx->kt->small_min_uses < 0) continue;
            memcpy(kk.b, keys_xy + 64 * (size_t)k, 64);
            auto sm = ctx->kt->small_map.find(kk);
            if (sm != ctx->kt->small_map.end()) {
                if (!touched) { ctx->kt->tick++; touched = true; }
                slot_of[k] = make_small_handle(ctx, sm->second); ctx->kt->small_tick[sm->second] = ctx->kt->tick; continue;
            }
            uint32_t total = uses[k];
            if (total < (uint32_t)ctx->kt->small_min_uses) {
                uint64_t h0, h1;
                memcpy(&h0, kk.b + 8, 8); memcpy(&h1, kk.b + 40, 8);
                const uint64_t tag = ((h0 * 0x9E3779B97F4A7C15ull) ^ (h1 * 0xC2B2AE3D27D4EB4Full)) | 1ull;
                const size_t b0 = (size_t)(tag >> 20) & (ctx->kt->seen_tag.size() - 1) & ~(size_t)3;   // bucket of four entries
                size_t at = b0, weakest = b0;
                bool found = false;
                for (size_t q = b0; q < b0 + 4 && !found; q++) {
                    if (ctx->kt->seen_tag[q] == tag) { at = q; found = true; }
                    else if (ctx->kt->seen_tag[q] == 0) { if (ctx->kt->seen_tag[weakest] != 0) weakest = q; }
                    else if (ctx->kt->seen_tag[weakest] != 0 && ctx->kt->seen_cnt[q] < ctx->kt->seen_cnt[weakest]) weakest = q;
                }
                if (!found) { at = weakest; ctx->kt->seen_tag[at] = tag; ctx->kt->seen_cnt[at] = 0; }      // an empty entry, else the least used one
                ctx->kt->seen_cnt[at] += uses[k];
                total = ctx->kt->seen_cnt[at];
                if (total >= (uint32_t)ctx->kt->small_min_uses) { ctx->kt->seen_tag[at] = 0; ctx->kt->seen_cnt[at] = 0; }
            }
            if (total >= (uint32_t)ctx->kt->small_min_uses) want_small.push_back(k);
        }
    }
    if (!want_big.empty() && (int)want_big.size() <= ctx->kt->key_slots) {
        std::vector<uint8_t> wk(64 * want_big.size());
        std::vector<int32_t> ws(want_big.size(), -1);
        for (size_t i = 0; i < want_big.size(); i++) memcpy(wk.data() + 64 * i, keys_xy + 64 * (size_t)want_big[i], 64);
        int rc = fabgpu_keys_register(ctx, wk.data(), (int)want_big.size(), ws.data());
        if (rc) return rc;
        for (size_t i = 0; i < want_big.size(); i++) slot_of[want_big[i]] = ws[i];
    } else if (ctx->kt->small_min_uses >= 0) {
        for (int k : want_big) want_small.push_back(k);              // more busy keys than big slots: the small tier takes them
    }
    if (!want_small.empty()) {
        std::vector<uint8_t> wk(64 * want_small.size());
        std::vector<int32_t> ws(want_small.size(), -1);
        for (size_t i = 0; i < want_small.size(); i++) memcpy(wk.data() + 64 * i, keys_xy + 64 * (size_t)want_small[i], 64);
        int rc = small_register(ctx, wk.data(), (int)want_small.size(), ws.data());
        if (rc) return rc;
        for (size_t i = 0; i < want_small.size(); i++) slot_of[want_small[i]] = ws[i];
    }
    return FABGPU_OK;
}

// Default: gates on the device (one context device; a multi-device context keeps the host-gated split).
static bool device_gates_apply(const fabgpu_ctx* ctx, const uint32_t* dig_off, const uint32_t* sig_off, size_t n)
{
    const char* dg = getenv("FABGPU_BCCSP_HOST_GATES");
    return !(dg && dg[0] == '1') && ctx->devs.size() == 1 && n > 0 && n < (1u << 27) && sig_off[n] < (1u << 31) && dig_off[n] < (1u << 31);
}

static int bccsp_batch_hostgated(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, const int32_t* key_idx, const uint8_t* digests,
                                 const uint32_t* dig_off, const uint8_t* sigs, const uint32_t* sig_off, size_t n, uint8_t* status,
                                 const std::vector<int32_t>& slot_of);

int fabgpu_bccsp_verify_batch_async(fabgpu_ctx* ctx, int slot, const uint8_t* keys_xy, int K, const int32_t* key_idx, const uint8_t* digests,
                                    const uint32_t* dig_off, const uint8_t* sigs, const uint32_t* sig_off, size_t n)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || (n && (!key_idx || !dig_off || !sig_off))) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->gb_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);       // host threads (staging pool) and the key cache: one submitter at a time
    auto& gb = ctx->gb[slot];
    if (gb.busy) { ctx->last_error = "slot already holds a batch: call fabgpu_bccsp_verify_batch_wait first"; return FABGPU_E_ARG; }
    auto t_start = std::chrono::steady_clock::now();
    ctx->timing[0] = ctx->timing[1] = ctx->timing[2] = ctx->timing[3] = 0;
    std::vector<int32_t> slot_of;
    int rc = resolve_key_tables(ctx, keys_xy, K, key_idx, n, slot_of);
    if (rc) return rc;
    ctx->timing[0] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_start).count();
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    gb.n = n;
    if (device_gates_apply(ctx, dig_off, sig_off, n)) {
        rc = bccsp_device_submit(ctx, slot, keys_xy, K, key_idx, digests, dig_off, sigs, sig_off, n, slot_of);
        if (rc) { cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get()); return rc; }
        gb.on_device = true;
    } else {
        // host-gated split (several devices, or FABGPU_BCCSP_HOST_GATES=1): it pipelines internally over both pinned SoA
        // slots, so it completes here and _wait only hands the statuses out
        gb.done_status.assign(n, 0);
        if (n) { rc = bccsp_batch_hostgated(ctx, keys_xy, K, key_idx, digests, dig_off, sigs, sig_off, n, gb.done_status.data(), slot_of); if (rc) return rc; }
        gb.on_device = false;
    }
    gb.busy = true;
    return FABGPU_OK;
}

int fabgpu_bccsp_batch_buffers(fabgpu_ctx* ctx, int slot, size_t n_cap, size_t sig_bytes_cap, size_t dig_bytes_cap, int k_cap, uint8_t** keys_xy,
                               int32_t** key_idx, uint8_t** digests, uint32_t** dig_off, uint8_t** sigs, uint32_t** sig_off)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || k_cap < 0 || !keys_xy || !key_idx || !digests || !dig_off || !sigs || !sig_off) return FABGPU_E_ARG;
    if (ctx->devs.size() != 1) { ctx->last_error = "the in-place batch form runs the gates on the device: single-device contexts only"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk(ctx->gb_mu[slot]);
    auto& gb = ctx->gb[slot];
    if (gb.busy) { ctx->last_error = "slot holds a batch in flight"; return FABGPU_E_ARG; }
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    int rc = gate_bufs_reserve(ctx, slot, n_cap, sig_bytes_cap, dig_bytes_cap, (size_t)k_cap);
    if (rc) return rc;
    *keys_xy = gb.h_keys.get(); *key_idx = gb.h_kidx.get(); *digests = gb.h_digs.get(); *dig_off = gb.h_dig_off.get(); *sigs = gb.h_sigs.get(); *sig_off = gb.h_sig_off.get();
    return FABGPU_OK;
}

int fabgpu_bccsp_verify_batch_inplace_async(fabgpu_ctx* ctx, int slot, int K, size_t n)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || K < 0) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->gb_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& gb = ctx->gb[slot];
    if (gb.busy) { ctx->last_error = "slot already holds a batch: call fabgpu_bccsp_verify_batch_wait first"; return FABGPU_E_ARG; }
    if (n > gb.n_cap() || (size_t)K > gb.k_cap() || !gb.h_sig_off.get()) { ctx->last_error = "batch exceeds the capacities given to fabgpu_bccsp_batch_buffers"; return FABGPU_E_ARG; }
    if (n && (gb.h_sig_off.get()[0] != 0 || gb.h_dig_off.get()[0] != 0 || gb.h_sig_off.get()[n] > gb.sig_cap() || gb.h_dig_off.get()[n] > gb.dig_cap())) {
        ctx->last_error = "offset tables must start at 0 and stay inside the buffers"; return FABGPU_E_ARG;
    }
    if (!device_gates_apply(ctx, gb.h_dig_off.get(), gb.h_sig_off.get(), n) && n) { ctx->last_error = "the in-place batch form needs the device gates"; return FABGPU_E_ARG; }
    auto t_start = std::chrono::steady_clock::now();
    ctx->timing[0] = ctx->timing[1] = ctx->timing[2] = ctx->timing[3] = 0;
    std::vector<int32_t> slot_of;
    int rc = resolve_key_tables(ctx, gb.h_keys.get(), K, gb.h_kidx.get(), n, slot_of);
    if (rc) return rc;
    ctx->timing[0] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_start).count();
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    gb.n = n;
    if (n) {
        rc = bccsp_device_submit(ctx, slot, gb.h_keys.get(), K, gb.h_kidx.get(), gb.h_digs.get(), gb.h_dig_off.get(), gb.h_sigs.get(), gb.h_sig_off.get(), n, slot_of, true);
        if (rc) { cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get()); return rc; }
        gb.on_device = true;
    } else { gb.done_status.clear(); gb.on_device = false; }
    gb.busy = true;
    return FABGPU_OK;
}

int fabgpu_bccsp_verify_batch_wait(fabgpu_ctx* ctx, int slot, uint8_t* status, size_t n)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->gb_mu[slot]);
    auto& gb = ctx->gb[slot];
    if (!gb.busy) { ctx->last_error = "no batch in flight on this slot"; return FABGPU_E_ARG; }
    if (n != gb.n || (n && !status)) { ctx->last_error = "status buffer does not match the submitted batch"; return FABGPU_E_ARG; }
    gb.busy = false;
    if (gb.on_device) return bccsp_device_finish(ctx, slot, status);
    if (n) memcpy(status, gb.done_status.data(), n);
    return FABGPU_OK;
}

int fabgpu_bccsp_verify_batch(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, const int32_t* key_idx, const uint8_t* digests,
                              const uint32_t* dig_off, const uint8_t* sigs, const uint32_t* sig_off, size_t n, uint8_t* status)
{
    if (!ctx || (n && (!status || !key_idx || !dig_off || !sig_off))) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->sync_mu);        // one synchronous caller at a time
    // A large call is cut into one chunk per slot: the copy of chunk c+1 runs under the kernels of chunk c and all chunks' verify
    // launches are resident together (they fill the machine like one launch).  Needs every slot free; otherwise, and for
    // small calls, the whole batch goes through slot 0.
    if (n >= 24576 && device_gates_apply(ctx, dig_off, sig_off, n)) {
        std::unique_lock<std::mutex> l[FABGPU_SLOTS];
        bool all_free = true;
        for (int c = 0; c < FABGPU_SLOTS; c++) { l[c] = std::unique_lock<std::mutex>(ctx->gb_mu[c]); all_free = all_free && !ctx->gb[c].busy; }
        if (all_free) {
            size_t lo[FABGPU_SLOTS + 1];
            for (int c = 0; c <= FABGPU_SLOTS; c++) lo[c] = n * (size_t)c / FABGPU_SLOTS;
            int submitted = 0, rc = FABGPU_OK;
            {
                std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
                auto t_start = std::chrono::steady_clock::now();
                ctx->timing[0] = ctx->timing[1] = ctx->timing[2] = ctx->timing[3] = 0;
                std::vector<int32_t> slot_of;
                rc = resolve_key_tables(ctx, keys_xy, K, key_idx, n, slot_of);
                ctx->timing[0] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_start).count();
                if (!rc && fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; rc = FABGPU_E_INJECTED; }
                for (int c = 0; c < FABGPU_SLOTS && !rc; c++) {
                    rc = bccsp_device_submit(ctx, c, keys_xy, K, key_idx + lo[c], digests, dig_off + lo[c], sigs, sig_off + lo[c], lo[c + 1] - lo[c], slot_of);
                    if (!rc) submitted++;
                }
            }
            for (int c = 0; c < submitted; c++) {                       // drain what was enqueued even after an error
                int rc2 = bccsp_device_finish(ctx, c, status + lo[c]);
                if (!rc) rc = rc2;
            }
            if (rc && submitted < FABGPU_SLOTS) cudaStreamSynchronize(ctx->devs[0].slot[submitted].stream.get());   // a submit that failed half-way
            return rc;
        }
    }
    int rc = fabgpu_bccsp_verify_batch_async(ctx, 0, keys_xy, K, key_idx, digests, dig_off, sigs, sig_off, n);
    if (rc) return rc;
    return fabgpu_bccsp_verify_batch_wait(ctx, 0, status, n);
}

// Host-gated form.  Gates run on the context's host threads; a signature that fails a gate keeps its position with
// r = s = 0 (the kernel rejects it at once) so that packing needs no compaction and stays parallel.
static int bccsp_batch_hostgated(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, const int32_t* key_idx, const uint8_t* digests,
                                 const uint32_t* dig_off, const uint8_t* sigs, const uint32_t* sig_off, size_t n, uint8_t* status,
                                 const std::vector<int32_t>& slot_of)
{
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::micro>(b - a).count();
    };
    // The call is cut into chunks that alternate between the two pinned slots: while the GPU works on one chunk the
    // host threads gate and pack the next, and the statuses of the chunk before are scattered.
    const int T = ctx->pool->size();
    size_t chunk = ctx->max_batch;
    if (n > 16384) {
        const char* ev = getenv("FABGPU_E2E_CHUNKS");
        const size_t parts = ev ? (size_t)std::max(1, atoi(ev)) : 4;
        chunk = std::min(ctx->max_batch, std::max((size_t)8192, round_up32((n + parts - 1) / parts)));
    }
    struct InFlight { bool active = false; size_t base = 0, cnt = 0; } fl[FABGPU_SLOTS];
    auto retire = [&](int sl) -> int {
        if (!fl[sl].active) return FABGPU_OK;
        auto a = now();
        int rc = fabgpu_wait(ctx, sl);
        auto b = now();
        ctx->timing[2] += us(a, b);
        if (rc) return rc;
        HostSlot& hsl = ctx->hslot[sl];
        const size_t base = fl[sl].base, cnt = fl[sl].cnt;
        ctx->pool->run([&](int tid) {
            const size_t lo = cnt * (size_t)tid / T, hi = cnt * (size_t)(tid + 1) / T;
            for (size_t k = lo; k < hi; k++) {
                if (status[base + k] != FABGPU_ST_VALID) continue;          // decided by a gate
                const bool ok = (hsl.h_mask.get()[k >> 5] >> (k & 31)) & 1u;
                const bool oc = (hsl.h_off.get()[k >> 5] >> (k & 31)) & 1u;
                status[base + k] = ok ? FABGPU_ST_VALID : (oc ? FABGPU_ST_ERR_OFF_CURVE : FABGPU_ST_INVALID);
            }
        });
        fl[sl].active = false;
        ctx->timing[3] += us(b, now());
        return FABGPU_OK;
    };
    int sl = 0;
    static const uint8_t kZero32[32] = {0};
    for (size_t base = 0; base < n; base += chunk, sl = (sl + 1) % FABGPU_SLOTS) {
        const size_t cnt = std::min(chunk, n - base);
        int rc = retire(sl);
        if (rc) return rc;
        HostSlot& hs = ctx->hslot[sl];
        std::atomic<size_t> asked{0};
        auto t0 = now();
        ctx->pool->run([&](int tid) {
            const size_t b = cnt * (size_t)tid / T, e = cnt * (size_t)(tid + 1) / T;
            size_t mine = 0;
            for (size_t k = b; k < e; k++) {
                const size_t i = base + k;
                const int32_t ki = key_idx[i];
                const size_t sl_ = sig_off[i + 1] - sig_off[i], dl = dig_off[i + 1] - dig_off[i];
                uint8_t st;
                if (ki < 0) st = FABGPU_ST_ERR_NIL_KEY;                    // bccsp/sw/impl.go:249-251
                else if (sl_ == 0) st = FABGPU_ST_ERR_EMPTY_SIG;           // :252-254
                else if (dl == 0) st = FABGPU_ST_ERR_EMPTY_DIGEST;         // :255-257
                else if (ki >= K || !keys_xy) st = FABGPU_ST_ERR_UNSUPPORTED_KEY;
                else {
                    host::Gate g;
                    host::gate_signature(sigs + sig_off[i], sl_, g, false);
                    st = (uint8_t)g.status;
                    if (g.status == FABGPU_ST_VALID) {
                        uint8_t ebuf[32];
                        host::hash_to_e(digests + dig_off[i], dl, ebuf);
                        // Qx / Qy are staged even for keys with a table: the handle is resolved again at enqueue time and, had
                        // the slot been recycled by then, the generic kernel verifies against these (never against stale bytes)
                        stage32(hs.h_in[0].get() + 32 * k, keys_xy + 64 * (size_t)ki);
                        stage32(hs.h_in[1].get() + 32 * k, keys_xy + 64 * (size_t)ki + 32);
                        stage32(hs.h_in[2].get() + 32 * k, ebuf);
                        stage32(hs.h_in[3].get() + 32 * k, g.r);
                        stage32(hs.h_in[4].get() + 32 * k, g.s);
                        mine++;
                    }
                }
                if (st != FABGPU_ST_VALID) { stage32(hs.h_in[3].get() + 32 * k, kZero32); stage32(hs.h_in[4].get() + 32 * k, kZero32); }
                stage_i32(hs.h_key_slot.get() + k, (st == FABGPU_ST_VALID) ? slot_of[ki] : -1);
                status[i] = st;
            }
            stage_fence();
            asked += mine;
        });
        auto t1 = now();
        ctx->timing[1] += us(t0, t1);
        if (asked.load() == 0) continue;
        rc = fabgpu_verify_p256_keyed_async(ctx, sl, cnt);
        if (rc) return rc;
        fl[sl].active = true; fl[sl].base = base; fl[sl].cnt = cnt;
        ctx->timing[2] += us(t1, now());
    }
    // drain in launch order
    for (int k = 0; k < FABGPU_SLOTS; k++, sl = (sl + 1) % FABGPU_SLOTS) {
        int rc = retire(sl);
        if (rc) return rc;
    }
    return FABGPU_OK;
}

void fabgpu_build_info(int* g_window_bits, int* key_window_bits)
{
    if (g_window_bits) *g_window_bits = FAB_WG;
    if (key_window_bits) *key_window_bits = FAB_WQ;
}

int fabgpu_last_timing(const fabgpu_ctx* ctx, double out_us[4])
{
    if (!ctx || !out_us) return FABGPU_E_ARG;
    for (int i = 0; i < 4; i++) out_us[i] = ctx->timing[i];
    return FABGPU_OK;
}

int fabgpu_bccsp_verify(fabgpu_ctx* ctx, const uint8_t* key_xy, const uint8_t* sig, size_t sig_len, const uint8_t* digest,
                        size_t digest_len, int* valid, char* err, size_t errcap)
{
    if (!ctx || !valid) return FABGPU_E_ARG;
    *valid = 0;
    std::string msg;
    auto finish = [&](const std::string& m) {
        if (err && errcap) { size_t k = std::min(errcap - 1, m.size()); memcpy(err, m.data(), k); err[k] = 0; }
        return FABGPU_OK;
    };
    // sw.CSP.Verify argument gates, reference bccsp/sw/impl.go:249-257
    if (!key_xy) return finish("Invalid Key. It must not be nil.");
    if (!sig || sig_len == 0) return finish("Invalid signature. Cannot be empty.");
    if (!digest || digest_len == 0) return finish("Invalid digest. Cannot be empty.");
    host::Gate g;
    host::gate_signature(sig, sig_len, g, true);
    if (g.status != FABGPU_ST_VALID && g.status != FABGPU_ST_INVALID)
        return finish("Failed verifing with opts [<nil>]: " + g.err);          // errors.Wrapf at impl.go:266
    if (g.status == FABGPU_ST_INVALID) return finish("");                       // r >= 2^256: (false, nil)
    uint8_t e[32];
    host::hash_to_e(digest, digest_len, e);
    uint32_t mask = 0, off = 0;
    int rc = fabgpu_verify_p256_host(ctx, key_xy, key_xy + 32, e, g.r, g.s, 1, &mask, &off);
    if (rc) return rc;
    if (off & 1u) { ctx->last_error = "public key is not on P-256"; return FABGPU_E_ARG; }
    *valid = (int)(mask & 1u);
    return finish("");
}

// ---- block-level pre-pass -------------------------------------------------------------------------------------------

// The MSP stream (fabgpu_ctx::MspAdmit), created on first use on device 0 of the context
static int msp_stream(fabgpu_ctx* ctx, cudaStream_t* out)
{
    auto& a = ctx->adm;
    if (!a.stream) {
        cudaStream_t st = nullptr; cudaEvent_t ev = nullptr;
        CK(ctx, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); a.stream.reset(st);
        CK(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); a.ev.reset(ev);
        for (auto& e : a.stage_ev) { cudaEvent_t x = nullptr; CK(ctx, cudaEventCreateWithFlags(&x, cudaEventDisableTiming)); e.reset(x); }
    }
    *out = a.stream.get();
    return FABGPU_OK;
}

// Raw table slots of identities [i0, i1) from their handles, and the classes they add (DevMsp::all_slots / classes)
static void msp_raw_slots(fabgpu_ctx* ctx, int i0, int i1, int32_t* raw)
{
    auto& dm = ctx->dm;
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::lock_guard<std::mutex> kl(ctx->kt->mu);
    for (int i = i0; i < i1; i++) {
        raw[i - i0] = handle_to_slot(ctx, ctx->identity_slot[i]);
        if (raw[i - i0] < 0) { dm.all_slots = false; dm.classes |= raw[i - i0] == -1 ? CLASS_GENERIC : CLASS_SMALL; }
    }
}

static int32_t msp_code_of(fabgpu_ctx* ctx, const std::string& mspid)
{
    auto& codes = ctx->dm.codes;
    auto it = codes.find(mspid);
    if (it != codes.end()) return it->second;
    const int32_t c = (int32_t)codes.size();
    codes[mspid] = c;
    return c;
}

// Device copy of the MSP view and the policy for block_plan_kernel / block_decide_kernel (device 0 of the context).
static int upload_msp(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* keys_xy, const uint8_t* valid, int n_ids,
                      const int32_t* policy_nodes, int n_nodes)
{
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t ms = nullptr;
    if (int rc = msp_stream(ctx, &ms)) return rc;
    // blocks already enqueued on a slot were launched with the OLD tables (passed by value), and admissions may still be copying into
    // them: let both finish before those go away
    for (auto& ds : ctx->devs[0].slot) CK(ctx, cudaStreamSynchronize(ds.stream.get()));
    CK(ctx, cudaStreamSynchronize(ms));
    dm = fabgpu_ctx::DevMsp();
    ctx->adm.admitted = ctx->adm.ev_set = false;
    ctx->kpt = bdev::KeyPolicyTable();                       // its SignedBy nodes index the principals being replaced
    // MSP-id codes: equal strings <=> equal codes, shared between identities and policy principals; kept for later admissions
    std::vector<int32_t> msp_code(n_ids > 0 ? n_ids : 1, -1), pcode(ctx->principals.size() ? ctx->principals.size() : 1, -1);
    for (int i = 0; i < n_ids; i++) msp_code[i] = msp_code_of(ctx, ctx->msp.mspid[i]);
    for (size_t i = 0; i < ctx->principals.size(); i++) pcode[i] = msp_code_of(ctx, ctx->principals[i]);
    dm.mirror.configure(id_blob, id_off, n_ids);
    const uint32_t hsz = dm.mirror.size();
    dm.all_slots = true;
    std::vector<int32_t> raw_slot(n_ids > 0 ? n_ids : 1, -1);
    dm.classes = 0;
    msp_raw_slots(ctx, 0, n_ids, raw_slot.data());
    auto up = [&](auto& dst, const void* src, size_t bytes) -> int {
        if (int rc = dst.reserve(ctx, bytes + 8)) return rc;   // slack: word-wise readers may touch the aligned word past the end
        if (bytes) CK(ctx, cudaMemcpy(dst.get(), src, bytes, cudaMemcpyHostToDevice));
        return FABGPU_OK;
    };
    auto up_ms = [&](auto& dst, const void* src, size_t bytes) -> int {
        if (int rc = msp_grow(ctx, dst, ms, bytes, 0)) return rc;
        if (bytes) CK(ctx, cudaMemcpyAsync(dst.get(), src, bytes, cudaMemcpyHostToDevice, ms));
        return FABGPU_OK;
    };
    const size_t blob_len = n_ids ? id_off[n_ids] : 0;
    if (up_ms(dm.id_blob, id_blob, blob_len) || up_ms(dm.id_off, id_off, 4 * (size_t)(n_ids + 1) * (n_ids ? 1 : 0)) || up_ms(dm.valid, valid, (size_t)n_ids) ||
        up_ms(dm.keys_xy, keys_xy, 64 * (size_t)n_ids) || up_ms(dm.key_slot, raw_slot.data(), 4 * (size_t)n_ids) ||
        up_ms(dm.msp_code, msp_code.data(), 4 * (size_t)n_ids) || up_ms(dm.ht_hash, dm.mirror.ht_hash.data(), 8 * (size_t)hsz) ||
        up_ms(dm.ht_idx, dm.mirror.ht_idx.data(), 4 * (size_t)hsz) ||
        up(dm.nodes, policy_nodes, 16 * (size_t)n_nodes) || up(dm.principal_code, pcode.data(), 4 * ctx->principals.size()) ||
        up(dm.channel, ctx->channel.data(), ctx->channel.size()))
        return FABGPU_E_CUDA;
    CK(ctx, cudaStreamSynchronize(ms));                      // the sources are the caller's and local vectors
    dm.ht_size = n_ids ? hsz : 0; dm.n_ids = n_ids; dm.n_nodes = n_nodes; dm.n_principals = (int32_t)ctx->principals.size();
    dm.channel_len = (uint32_t)ctx->channel.size();
    dm.configured = true;
    return FABGPU_OK;
}


// Small tables for identities: every identity gets a small table; the ones whose key ALREADY owns a window table -- the integrator
// registered the few busy ones (the endorsing peers) with fabgpu_keys_register beforehand -- keep using that.  The tier of an MSP with more
// identities than window-table slots, and of every admitted identity.
static int msp_small_tier(fabgpu_ctx* ctx, const uint8_t* keys_xy, int n_ids, int32_t* handles)
{
    int rc = small_register(ctx, keys_xy, n_ids, handles);
    if (rc) return rc;
    std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->kt->key_map.empty()) return FABGPU_OK;
    std::string kbuf(64, '\0');
    for (int i = 0; i < n_ids; i++) {
        memcpy(&kbuf[0], keys_xy + 64 * (size_t)i, 64);
        auto it = ctx->kt->key_map.find(kbuf);
        if (it != ctx->kt->key_map.end()) handles[i] = make_handle(ctx, it->second);
    }
    return FABGPU_OK;
}

// Height of node i's tree (a leaf is 0), or -1 when it is deeper than BD_MAX_POLICY_DEPTH or runs into a cycle (a cycle makes the
// path longer than any bound).  height: memo, -1 = not known yet.  The path length bounds the recursion.
static int policy_height(const std::vector<blockval::PolicyNode>& nodes, int i, int path, std::vector<int>& height)
{
    if (path > BD_MAX_POLICY_DEPTH) return -1;
    if (height[i] >= 0) return height[i];
    int h = 0;
    if (nodes[i].type == 0 || nodes[i].type == 2)
        for (int c = nodes[i].first_child; c < nodes[i].first_child + nodes[i].n_children; c++) {
            const int hc = policy_height(nodes, c, path + 1, height);
            if (hc < 0 || hc + 1 > BD_MAX_POLICY_DEPTH) return -1;
            h = std::max(h, hc + 1);
        }
    return height[i] = h;
}

// What eval_policy can evaluate exactly: node types 0 (NOutOf), 1 (SignedBy) and 2 (ImplicitMeta), children inside the array,
// SignedBy indices inside the principals, and from every node a tree at most BD_MAX_POLICY_DEPTH deep without cycles.  Past that
// depth the device would report ENDORSEMENT_POLICY_FAILURE where the reference, which has no depth limit, may accept: such a
// policy is refused, and the caller validates on the CPU.  ImplicitMeta nodes must be what NewImplicitMetaPolicy builds
// (implicitmeta.go:44-58): a threshold in [1, n_children], or 0 over no children; and never a child of an NOutOf node, since a
// signature policy compiles only NOutOf and SignedBy (cauthdsl.go:24-92).
static const char* check_policy(const std::vector<blockval::PolicyNode>& nodes, int n_principals)
{
    const int64_t n_nodes = (int64_t)nodes.size();
    for (const auto& nd : nodes) {
        if (nd.type < 0 || nd.type > 2) return "policy node type is not NOutOf (0), SignedBy (1) or ImplicitMeta (2)";
        if (nd.type != 1 && (nd.first_child < 0 || nd.n_children < 0 || (int64_t)nd.first_child + nd.n_children > n_nodes))
            return "policy node children out of range";
        if (nd.type == 1 && (nd.n < 0 || nd.n >= n_principals)) return "SignedBy principal index out of range";
        if (nd.type == 2 && !(nd.n >= 1 ? nd.n <= nd.n_children : nd.n == 0 && nd.n_children == 0))
            return "ImplicitMeta threshold outside [1, n_children] (or 0 with no children)";
    }
    for (const auto& nd : nodes)
        if (nd.type == 0)
            for (int c = nd.first_child; c < nd.first_child + nd.n_children; c++)
                if (nodes[c].type == 2) return "ImplicitMeta node below an NOutOf node";
    std::vector<int> height(nodes.size(), -1);
    for (int i = 0; i < (int)n_nodes; i++)
        if (policy_height(nodes, i, 0, height) < 0) return "policy tree deeper than the device evaluates, or cyclic";
    return nullptr;
}

int fabgpu_msp_configure(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob,
                         const uint32_t* mspid_off, const uint8_t* keys_xy, const uint8_t* valid, int n_ids,
                         const int32_t* policy_nodes, int n_nodes, const uint8_t* principal_blob, const uint32_t* principal_off,
                         int n_principals, const char* channel_id)
{
    if (!ctx || n_ids < 0 || n_nodes < 0 || n_principals < 0 || !channel_id) return FABGPU_E_ARG;
    if (n_ids && (!id_blob || !id_off || !mspid_blob || !mspid_off || !keys_xy || !valid)) return FABGPU_E_ARG;
    if (n_nodes && !policy_nodes) return FABGPU_E_ARG;
    {
        std::vector<blockval::PolicyNode> nodes;
        for (int i = 0; i < n_nodes; i++)
            nodes.push_back({policy_nodes[4 * i], policy_nodes[4 * i + 1], policy_nodes[4 * i + 2], policy_nodes[4 * i + 3]});
        if (const char* err = check_policy(nodes, n_principals)) { ctx->last_error = err; return FABGPU_E_ARG; }
    }
    {
        std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
        ctx->msp = blockval::MspTable();
        for (int i = 0; i < n_ids; i++) {
            ctx->msp.add(id_blob + id_off[i], id_off[i + 1] - id_off[i]);
            ctx->msp.mspid.emplace_back((const char*)mspid_blob + mspid_off[i], mspid_off[i + 1] - mspid_off[i]);
        }
        ctx->msp.keys_xy.assign(keys_xy, keys_xy + 64 * (size_t)n_ids);
        ctx->msp.valid.assign(valid, valid + n_ids);
        ctx->policy.clear();
        for (int i = 0; i < n_nodes; i++)
            ctx->policy.push_back({policy_nodes[4 * i], policy_nodes[4 * i + 1], policy_nodes[4 * i + 2], policy_nodes[4 * i + 3]});
        ctx->principals.clear();
        for (int i = 0; i < n_principals; i++)
            ctx->principals.emplace_back((const char*)principal_blob + principal_off[i], principal_off[i + 1] - principal_off[i]);
        ctx->channel = channel_id;
        ctx->identity_slot.assign(n_ids, -1);
        ctx->identity_tier.assign(n_ids, n_ids <= ctx->kt->key_slots ? TIER_WINDOW : TIER_SMALL);
    }
    // identities are long-lived: give every key a table now (what KeyImport does when the MSP deserialises an identity)
    // An MSP with more identities than big-table slots (client certificates) puts them in the small tier instead.
    if (n_ids > 0 && n_ids <= ctx->kt->key_slots) {
        int rc = fabgpu_keys_register(ctx, keys_xy, n_ids, ctx->identity_slot.data());
        if (rc) return rc;
    } else if (n_ids > 0) {
        int rc = msp_small_tier(ctx, keys_xy, n_ids, ctx->identity_slot.data());      // also with the small tier off or too small: pre-registered window tables are still picked up
        if (rc) return rc;
    }
    return upload_msp(ctx, id_blob, id_off, keys_xy, valid, n_ids, policy_nodes, n_nodes);
}

// drains the block slots' streams and the MSP stream: kernels already enqueued keep reading the tables they were launched with
static int drain_block_streams(fabgpu_ctx* ctx)
{
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    for (auto& ds : ctx->devs[0].slot) CK(ctx, cudaStreamSynchronize(ds.stream.get()));
    if (ctx->adm.stream) CK(ctx, cudaStreamSynchronize(ctx->adm.stream.get()));
    return FABGPU_OK;
}

int fabgpu_msp_identity_groups(fabgpu_ctx* ctx, const int32_t* group, int n_ids)
{
    if (!ctx || n_ids < 0 || (n_ids && !group)) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    if (n_ids != dm.n_ids) { ctx->last_error = "group table does not match the identities the MSP table holds"; return FABGPU_E_ARG; }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.group = {};
    if (n_ids == 0) return FABGPU_OK;
    cudaStream_t ms = nullptr;
    if ((rc = msp_stream(ctx, &ms)) || (rc = msp_grow(ctx, dm.group, ms, 4 * (size_t)n_ids, 0))) return rc;
    CK(ctx, cudaMemcpyAsync(dm.group.get(), group, 4 * (size_t)n_ids, cudaMemcpyHostToDevice, ms));
    CK(ctx, cudaStreamSynchronize(ms));
    return FABGPU_OK;
}

int fabgpu_msp_principal_bits(fabgpu_ctx* ctx, const uint32_t* bits, int n_ids, int n_principals)
{
    if (!ctx || n_ids < 0 || n_principals < 0 || (n_ids && !bits)) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    if (n_ids && (n_ids != dm.n_ids || n_principals != dm.n_principals)) {
        ctx->last_error = "principal bits do not match the identities the MSP table holds and the principals given to fabgpu_msp_configure";
        return FABGPU_E_ARG;
    }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.pbits = {}; dm.pbits_words = 0;
    if (n_ids == 0) return FABGPU_OK;
    const int W = (n_principals + 31) / 32;
    const size_t bytes = 4 * (size_t)n_ids * W;
    cudaStream_t ms = nullptr;
    if ((rc = msp_stream(ctx, &ms)) || (rc = msp_grow(ctx, dm.pbits, ms, bytes, 0))) return rc;     // non-null even with no principals: it selects the bit test
    if (bytes) CK(ctx, cudaMemcpyAsync(dm.pbits.get(), bits, bytes, cudaMemcpyHostToDevice, ms));
    CK(ctx, cudaStreamSynchronize(ms));
    dm.pbits_words = W;
    return FABGPU_OK;
}

// A failed admission may have left the device table half written: from here on no lookup finds an identity (every transaction is 254)
// until fabgpu_msp_configure installs a table again.  The host's per-identity state goes back to the n0 identities the device arrays
// are known to hold, so that the stale-handle re-issue in block_submit never writes past them.
static int msp_admit_fail(fabgpu_ctx* ctx, int rc, int n0)
{
    ctx->dm.ht_size = 0; ctx->dm.configured = false;
    ctx->identity_slot.resize(n0); ctx->identity_tier.resize(n0);
    ctx->msp.serialized.resize(n0); ctx->msp.mspid.resize(n0); ctx->msp.keys_xy.resize(64 * (size_t)n0); ctx->msp.valid.resize(n0);
    ctx->last_error += " (the MSP table is lost until fabgpu_msp_configure installs one)";
    return rc;
}

int fabgpu_msp_identities_add(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob, const uint32_t* mspid_off,
                              const uint8_t* keys_xy, const uint8_t* valid, const int32_t* group, const uint32_t* bits, int n)
{
    if (!ctx) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm; auto& a = ctx->adm;
    if (!dm.configured) { ctx->last_error = "no MSP table: call fabgpu_msp_configure first"; return FABGPU_E_ARG; }
    if (const char* err = dm.mirror.check_add(id_blob, id_off, mspid_blob, mspid_off, keys_xy, valid, group, bits, n, dm.group.get() != nullptr,
                                              dm.pbits.get() != nullptr)) {
        ctx->last_error = err; return FABGPU_E_ARG;
    }
    if (n > INT32_MAX - dm.n_ids) { ctx->last_error = "too many identities"; return FABGPU_E_ARG; }
    if (n == 0) return FABGPU_OK;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t ms = nullptr;
    if (int rc = msp_stream(ctx, &ms)) return rc;
    // key tables first: nothing of the table has changed if this fails
    std::vector<int32_t> handles(n, -1);
    if (int rc = msp_small_tier(ctx, keys_xy, n, handles.data())) return rc;
    const int n0 = dm.n_ids, n1 = n0 + n;
    const size_t W = (size_t)dm.pbits_words;
    // host side: the mirrors, the MSP-id codes and the new index slots
    ctx->identity_slot.insert(ctx->identity_slot.end(), handles.begin(), handles.end());
    ctx->identity_tier.resize(n1, TIER_SMALL);
    std::vector<int32_t> raw(n), code(n);
    msp_raw_slots(ctx, n0, n1, raw.data());
    for (int i = 0; i < n; i++) {
        std::string mspid((const char*)mspid_blob + mspid_off[i], mspid_off[i + 1] - mspid_off[i]);
        code[i] = msp_code_of(ctx, mspid);
        ctx->msp.add(id_blob + id_off[i], id_off[i + 1] - id_off[i]);
        ctx->msp.mspid.push_back(std::move(mspid));
    }
    ctx->msp.keys_xy.insert(ctx->msp.keys_xy.end(), keys_xy, keys_xy + 64 * (size_t)n);
    ctx->msp.valid.insert(ctx->msp.valid.end(), valid, valid + n);
    const size_t blob0 = dm.mirror.blob.size();
    std::vector<uint32_t> dirty;
    const bool full = dm.mirror.add(id_blob, id_off, n, dirty);
    const uint32_t hsz = dm.mirror.size();
    // One pinned staging buffer: the appended rows, then the index (whole, or the changed slots: position, hash, identity).  Offsets
    // from n0 + 1 (from 0 for an empty table, whose array holds no offset yet).
    const size_t D = full ? hsz : dirty.size(), B = dm.mirror.blob.size() - blob0, f0 = n0 ? (size_t)n0 + 1 : 0, F = (size_t)n1 + 1 - f0;
    size_t at = 0;
    auto sec = [&](size_t bytes) { const size_t o = at; at += (bytes + 7) & ~(size_t)7; return o; };
    const size_t o_blob = sec(B), o_off = sec(4 * F), o_valid = sec(n), o_keys = sec(64 * (size_t)n), o_slot = sec(4 * (size_t)n),
                 o_code = sec(4 * (size_t)n), o_group = sec(group ? 4 * (size_t)n : 0), o_bits = sec(bits ? 4 * W * n : 0),
                 o_idx = sec(4 * D), o_hash = sec(8 * D), o_pos = sec(full ? 0 : 4 * D);
    const size_t o_scatter = o_idx;                                  // the scatter's values, copied to the device as one range
    const int r = (int)(a.seq++ % fabgpu_ctx::MspAdmit::RING);
    auto& hs = a.h_stage[r];
    if (a.stage_set[r]) CK(ctx, cudaEventSynchronize(a.stage_ev[r].get()));         // its copies, RING admissions ago
    if (at > hs.bytes())
        if (int rc = hs.reserve(ctx, std::max(at, 2 * hs.bytes()))) return msp_admit_fail(ctx, rc, n0);
    uint8_t* h = hs.get();
    memcpy(h + o_blob, dm.mirror.blob.data() + blob0, B);
    memcpy(h + o_off, dm.mirror.off.data() + f0, 4 * F);
    memcpy(h + o_valid, valid, n);
    memcpy(h + o_keys, keys_xy, 64 * (size_t)n);
    memcpy(h + o_slot, raw.data(), 4 * (size_t)n);
    memcpy(h + o_code, code.data(), 4 * (size_t)n);
    if (group) memcpy(h + o_group, group, 4 * (size_t)n);
    if (bits) memcpy(h + o_bits, bits, 4 * W * n);
    for (size_t d = 0; d < D; d++) {
        const uint32_t pos = full ? (uint32_t)d : dirty[d];
        if (!full) memcpy(h + o_pos + 4 * d, &pos, 4);
        memcpy(h + o_hash + 8 * d, &dm.mirror.ht_hash[pos], 8);
        memcpy(h + o_idx + 4 * d, &dm.mirror.ht_idx[pos], 4);
    }
    // 1. before the waits, what no block in flight reads: grown arrays (the old ones retired until after the waits), the appended rows
    //    past n0, a new index after growth, and the scatter's values.  The staging buffer's event follows these copies only.
    std::vector<void*> retired;
    uint8_t* d = nullptr;
    auto retire_all = [&] { for (void* q : retired) cudaFreeAsync(q, ms); retired.clear(); if (d) cudaFreeAsync(d, ms); d = nullptr; };
    auto fail = [&](int rc, const char* what) {
        if (what) ctx->last_error = what;
        for (auto& ds : ctx->devs[0].slot) cudaStreamSynchronize(ds.stream.get());     // the retired arrays' readers, before their free
        retire_all();
        return msp_admit_fail(ctx, rc, n0);
    };
    int rc = FABGPU_OK;
    if ((rc = msp_grow(ctx, dm.id_blob, ms, blob0 + B, blob0, &retired)) ||
        (rc = msp_grow(ctx, dm.id_off, ms, 4 * ((size_t)n1 + 1), 4 * f0, &retired)) ||
        (rc = msp_grow(ctx, dm.valid, ms, n1, n0, &retired)) || (rc = msp_grow(ctx, dm.keys_xy, ms, 64 * (size_t)n1, 64 * (size_t)n0, &retired)) ||
        (rc = msp_grow(ctx, dm.key_slot, ms, 4 * (size_t)n1, 4 * (size_t)n0, &retired)) ||
        (rc = msp_grow(ctx, dm.msp_code, ms, 4 * (size_t)n1, 4 * (size_t)n0, &retired)) ||
        (group && (rc = msp_grow(ctx, dm.group, ms, 4 * (size_t)n1, 4 * (size_t)n0, &retired))) ||
        (bits && (rc = msp_grow(ctx, dm.pbits, ms, 4 * W * n1, 4 * W * n0, &retired))) ||
        (full && ((rc = msp_grow(ctx, dm.ht_hash, ms, 8 * (size_t)hsz, 0, &retired, true)) ||
                  (rc = msp_grow(ctx, dm.ht_idx, ms, 4 * (size_t)hsz, 0, &retired, true)))))
        return fail(rc, nullptr);
    auto up = [&](void* dst, size_t o, size_t bytes) { return !bytes || cudaMemcpyAsync(dst, h + o, bytes, cudaMemcpyHostToDevice, ms) == cudaSuccess; };
    bool ok = up(dm.id_blob.get() + blob0, o_blob, B) && up(dm.id_off.get() + f0, o_off, 4 * F) && up(dm.valid.get() + n0, o_valid, n) &&
              up(dm.keys_xy.get() + 64 * (size_t)n0, o_keys, 64 * (size_t)n) && up(dm.key_slot.get() + n0, o_slot, 4 * (size_t)n) &&
              up(dm.msp_code.get() + n0, o_code, 4 * (size_t)n) && (!group || up(dm.group.get() + n0, o_group, 4 * (size_t)n)) &&
              (!bits || up(dm.pbits.get() + W * n0, o_bits, 4 * W * n));
    if (ok && full) ok = up(dm.ht_hash.get(), o_hash, 8 * D) && up(dm.ht_idx.get(), o_idx, 4 * D);
    if (ok && !full && D) {
        ok = cudaMallocAsync(reinterpret_cast<void**>(&d), at - o_scatter, ms) == cudaSuccess;
        if (!ok) d = nullptr;
        ok = ok && up(d, o_scatter, at - o_scatter);
    }
    ok = ok && cudaEventRecord(a.stage_ev[r].get(), ms) == cudaSuccess;
    if (!ok) return fail(FABGPU_E_CUDA, "MSP table admission copy failed");
    a.stage_set[r] = true;
    // 2. the MSP stream waits for every slot's last decide stage: a slot whose last block recorded none waits for all its stream holds
    auto& tx = ctx->txid;
    for (int k = 0; k < FABGPU_SLOTS && ok; k++) {
        if (!tx.decide_ev[k]) { cudaEvent_t ev = nullptr; ok = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess; tx.decide_ev[k].reset(ev); }
        if (ok && !tx.decide_set[k]) ok = cudaEventRecord(tx.decide_ev[k].get(), ctx->devs[0].slot[k].stream.get()) == cudaSuccess;
        ok = ok && cudaStreamWaitEvent(ms, tx.decide_ev[k].get(), 0) == cudaSuccess;
    }
    // 3. after them: the index slots blocks in flight read, in place, and the frees of what they were launched with
    if (ok && !full && D) {
        bdev::msp_scatter_kernel<<<(unsigned)((D + 255) / 256), 256, 0, ms>>>(dm.ht_hash.get(), dm.ht_idx.get(), reinterpret_cast<const uint32_t*>(d + (o_pos - o_scatter)),
                                                                               reinterpret_cast<const uint64_t*>(d + (o_hash - o_scatter)),
                                                                               reinterpret_cast<const int32_t*>(d), (uint32_t)D);
        ctx->launches++;
        ok = cudaGetLastError() == cudaSuccess;
    }
    if (!ok) return fail(FABGPU_E_CUDA, "MSP table admission enqueue failed");
    retire_all();
    CK(ctx, cudaEventRecord(a.ev.get(), ms));
    a.ev_set = a.admitted = true;
    dm.n_ids = n1; dm.ht_size = hsz;
    return FABGPU_OK;
}

int fabgpu_namespace_policies(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const int32_t* ns_root, int n_ns)
{
    if (!ctx || n_ns < 0 || (n_ns && (!ns_blob || !ns_off || !ns_root))) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    for (int i = 0; i < n_ns; i++)
        if (ns_root[i] < 0 || ns_root[i] >= dm.n_nodes || ns_off[i] > ns_off[i + 1]) { ctx->last_error = "namespace policy root out of range"; return FABGPU_E_ARG; }
    if (const char* err = capability::check_namespace_table(dm.mode == BD_MODE_V13, ctx->policy, ns_root, n_ns)) { ctx->last_error = err; return FABGPU_E_ARG; }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.ns_blob = {}; dm.ns_off = {}; dm.ns_root = {}; dm.n_ns = 0; dm.ns_root_host.clear();
    dm.ver_blob = {}; dm.ver_off = {};                                // versions name the entries of the table being replaced
    if (n_ns == 0) return FABGPU_OK;
    const size_t bl = ns_off[n_ns];
    if ((rc = dm.ns_blob.reserve(ctx, bl + 8))) return rc;
    if (bl) CK(ctx, cudaMemcpy(dm.ns_blob.get(), ns_blob, bl, cudaMemcpyHostToDevice));
    if ((rc = dm.ns_off.reserve(ctx, 4 * (size_t)(n_ns + 1)))) return rc;
    CK(ctx, cudaMemcpy(dm.ns_off.get(), ns_off, 4 * (size_t)(n_ns + 1), cudaMemcpyHostToDevice));
    if ((rc = dm.ns_root.reserve(ctx, 4 * (size_t)n_ns))) return rc;
    CK(ctx, cudaMemcpy(dm.ns_root.get(), ns_root, 4 * (size_t)n_ns, cudaMemcpyHostToDevice));
    dm.n_ns = n_ns; dm.ns_root_host.assign(ns_root, ns_root + n_ns);
    return FABGPU_OK;
}

int fabgpu_channel_capability(fabgpu_ctx* ctx, int cap)
{
    if (!ctx) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    if (const char* err = capability::check_capability(cap, ctx->policy, dm.ns_root_host.data(), dm.n_ns)) { ctx->last_error = err; return FABGPU_E_ARG; }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.mode = cap == FABGPU_CAP_V1_3 ? BD_MODE_V13 : BD_MODE_V20;
    return FABGPU_OK;
}

int fabgpu_namespace_versions(fabgpu_ctx* ctx, const uint8_t* ver_blob, const uint32_t* ver_off, int n_ns)
{
    if (!ctx || n_ns < 0 || (n_ns && (!ver_blob || !ver_off))) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    if (const char* err = capability::check_versions(ver_off, n_ns, dm.n_ns)) { ctx->last_error = err; return FABGPU_E_ARG; }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.ver_blob = {}; dm.ver_off = {};
    if (n_ns == 0) return FABGPU_OK;
    if ((rc = dm.ver_blob.reserve(ctx, ver_off[n_ns] + 8))) return rc;   // slack: bytes_equal reads whole aligned words
    if (ver_off[n_ns]) CK(ctx, cudaMemcpy(dm.ver_blob.get(), ver_blob, ver_off[n_ns], cudaMemcpyHostToDevice));
    if ((rc = dm.ver_off.reserve(ctx, 4 * (size_t)(n_ns + 1)))) { dm.ver_blob = {}; return rc; }
    if (cudaMemcpy(dm.ver_off.get(), ver_off, 4 * (size_t)(n_ns + 1), cudaMemcpyHostToDevice) != cudaSuccess) {
        dm.ver_blob = {}; dm.ver_off = {}; ctx->last_error = "namespace version upload failed"; return FABGPU_E_CUDA;
    }
    return FABGPU_OK;
}

int fabgpu_collection_policies(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                               const int32_t* coll_root, int n)
{
    if (!ctx || n < 0) return FABGPU_E_ARG;
    if (n && (!ns_blob || !ns_off || !coll_blob || !coll_off || !coll_root)) { ctx->last_error = "collection policy arrays missing"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    for (int i = 0; i < n; i++) {
        const char* err = coll_root[i] < 0 || coll_root[i] >= dm.n_nodes ? "collection policy root out of range"
                        : ns_off[i] > ns_off[i + 1] || coll_off[i] > coll_off[i + 1] ? "collection policy offsets decrease"
                        : coll_off[i] == coll_off[i + 1] ? "collection policy with an empty collection name" : nullptr;
        if (err) { ctx->last_error = err; return FABGPU_E_ARG; }
    }
    uint32_t size = 8; while (size < (uint32_t)(2 * n + 8)) size <<= 1;      // load factor <= 1/2
    std::vector<uint64_t> hh(size, 0); std::vector<int32_t> hi(size, -1);
    if (!bdev::coll_table_fill(ns_blob, ns_off, coll_blob, coll_off, n, size, hh.data(), hi.data())) {
        ctx->last_error = "collection policy given twice for one (namespace, collection)"; return FABGPU_E_ARG;
    }
    int rc = drain_block_streams(ctx); if (rc) return rc;
    dm.cp_ns_blob = {}; dm.cp_name_blob = {}; dm.cp_ns_off = {}; dm.cp_name_off = {}; dm.cp_root = {}; dm.cp_idx = {}; dm.cp_hash = {}; dm.cp_size = 0;
    if (n == 0) return FABGPU_OK;
    auto up = [&](auto& dst, const void* src, size_t bytes) -> int {
        if (int r = dst.reserve(ctx, bytes + 8)) return r;          // slack: bytes_equal reads whole aligned words
        if (bytes) CK(ctx, cudaMemcpy(dst.get(), src, bytes, cudaMemcpyHostToDevice));
        return FABGPU_OK;
    };
    if ((rc = up(dm.cp_ns_blob, ns_blob, ns_off[n])) || (rc = up(dm.cp_ns_off, ns_off, 4 * (size_t)(n + 1))) ||
        (rc = up(dm.cp_name_blob, coll_blob, coll_off[n])) || (rc = up(dm.cp_name_off, coll_off, 4 * (size_t)(n + 1))) ||
        (rc = up(dm.cp_root, coll_root, 4 * (size_t)n)) || (rc = up(dm.cp_hash, hh.data(), 8 * (size_t)size)) || (rc = up(dm.cp_idx, hi.data(), 4 * (size_t)size)))
        return rc;
    dm.cp_size = size;
    return FABGPU_OK;
}

// Brings the device copy of the key policy table up to ctx->kpt after a call changed it: the whole table after a rebuild, else the
// changed slots (scattered by kp_scatter_kernel), the new entry bytes and the new nodes.  Arrays grow by doubling, so an update costs
// what it changed.
static int kp_upload(fabgpu_ctx* ctx)
{
    auto& dm = ctx->dm; auto& k = ctx->kpt;
    if (!k.installed()) { dm.kp_slots = {}; dm.kp_blob = {}; dm.kp_val = {}; dm.kp_idx = {}; dm.kp_size = 0; dm.kp_n_nodes = 0; return FABGPU_OK; }
    dm.kp_size = 0;                                              // until the copy is complete
    auto grown = [](size_t need, size_t have) { return need <= have ? have : std::max(need, 2 * have); };
    // nodes: the configured ones, then the table's
    const size_t cfg = 16 * (size_t)dm.n_nodes, tail = 4 * k.nodes.size();
    if (k.full || cfg + tail + 8 > dm.nodes.bytes()) {
        std::vector<int32_t> all;
        for (const auto& nd : ctx->policy) { all.push_back(nd.type); all.push_back(nd.n); all.push_back(nd.first_child); all.push_back(nd.n_children); }
        all.insert(all.end(), k.nodes.begin(), k.nodes.end());
        if (int rc = dm.nodes.reserve(ctx, grown(cfg + tail + 8, dm.nodes.bytes()))) return rc;
        if (!all.empty()) CK(ctx, cudaMemcpy(dm.nodes.get(), all.data(), 4 * all.size(), cudaMemcpyHostToDevice));
    } else if (k.nodes.size() > k.nodes_from) {
        CK(ctx, cudaMemcpy(reinterpret_cast<uint8_t*>(dm.nodes.get()) + cfg + 4 * k.nodes_from, k.nodes.data() + k.nodes_from,
                           4 * (k.nodes.size() - k.nodes_from), cudaMemcpyHostToDevice));
    }
    // entry bytes (slack: bytes_equal reads whole aligned words)
    if (k.full || k.blob.size() + 8 > dm.kp_blob.bytes()) {
        if (int rc = dm.kp_blob.reserve(ctx, grown(k.blob.size() + 8, dm.kp_blob.bytes()))) return rc;
        if (!k.blob.empty()) CK(ctx, cudaMemcpy(dm.kp_blob.get(), k.blob.data(), k.blob.size(), cudaMemcpyHostToDevice));
    } else if (k.blob.size() > k.blob_from) {
        CK(ctx, cudaMemcpy(dm.kp_blob.get() + k.blob_from, k.blob.data() + k.blob_from, k.blob.size() - k.blob_from, cudaMemcpyHostToDevice));
    }
    // slots
    const size_t sb = sizeof(bdev::KpSlot) * k.slots.size();
    if (k.full || dm.kp_slots.bytes() != sb) {
        dm.kp_slots = {};
        if (int rc = dm.kp_slots.reserve(ctx, sb)) return rc;
        CK(ctx, cudaMemcpy(dm.kp_slots.get(), k.slots.data(), sb, cudaMemcpyHostToDevice));
    } else if (!k.dirty.empty()) {
        const size_t n = k.dirty.size();
        std::vector<bdev::KpSlot> val(n);
        for (size_t i = 0; i < n; i++) val[i] = k.slots[k.dirty[i]];
        if (int rc = dm.kp_idx.reserve(ctx, grown(4 * n, dm.kp_idx.bytes()))) return rc;
        if (int rc = dm.kp_val.reserve(ctx, grown(sizeof(bdev::KpSlot) * n, dm.kp_val.bytes()))) return rc;
        CK(ctx, cudaMemcpy(dm.kp_idx.get(), k.dirty.data(), 4 * n, cudaMemcpyHostToDevice));
        CK(ctx, cudaMemcpy(dm.kp_val.get(), val.data(), sizeof(bdev::KpSlot) * n, cudaMemcpyHostToDevice));
        bdev::kp_scatter_kernel<<<(unsigned)((n + 255) / 256), 256>>>(dm.kp_slots.get(), dm.kp_idx.get(), dm.kp_val.get(), (uint32_t)n);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaDeviceSynchronize());
    }
    dm.kp_size = (uint32_t)k.slots.size(); dm.kp_n_nodes = k.n_nodes();
    return FABGPU_OK;
}

static int key_policies(fabgpu_ctx* ctx, bool replace, const int32_t* nodes, int n_nodes, const uint8_t* ns_blob, const uint32_t* ns_off,
                        const uint8_t* coll_blob, const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off, const int32_t* root, int n)
{
    if (!ctx) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& dm = ctx->dm;
    int rc = drain_block_streams(ctx); if (rc) return rc;
    // a refused call leaves the table as it was (apply checks everything before it changes anything)
    if (const char* err = ctx->kpt.apply(replace, dm.n_nodes, dm.n_principals, nodes, n_nodes, ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, root, n)) {
        ctx->last_error = err; return FABGPU_E_ARG;
    }
    if ((rc = kp_upload(ctx))) {
        // A failed copy removes the table.  The node array also holds the configured policies, and growing it frees it first: put
        // those back, and if even that fails, refuse blocks until fabgpu_msp_configure installs them again.
        const std::string err = ctx->last_error;
        ctx->kpt = bdev::KeyPolicyTable(); dm.kp_size = 0; dm.kp_n_nodes = 0;
        std::vector<int32_t> cfg;
        for (const auto& nd : ctx->policy) { cfg.push_back(nd.type); cfg.push_back(nd.n); cfg.push_back(nd.first_child); cfg.push_back(nd.n_children); }
        const size_t bytes = 4 * cfg.size();
        dm.nodes_lost = !(bytes + 8 <= dm.nodes.bytes() || dm.nodes.reserve(ctx, bytes + 8) == FABGPU_OK) ||
                        (bytes && cudaMemcpy(dm.nodes.get(), cfg.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess);
        ctx->last_error = err;
    }
    return rc;
}

int fabgpu_key_policies(fabgpu_ctx* ctx, const int32_t* nodes, int n_nodes, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob,
                        const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off, const int32_t* root, int n)
{
    return key_policies(ctx, true, nodes, n_nodes, ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, root, n);
}

int fabgpu_key_policies_update(fabgpu_ctx* ctx, const int32_t* nodes, int n_nodes, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob,
                               const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off, const int32_t* root, int n)
{
    return key_policies(ctx, false, nodes, n_nodes, ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, root, n);
}

// ---- committed tx-id set (fabgpu_committed_txids / _add / _info); every step below runs under slot0_mu -----------------------------
// Brings the set's stream behind every block already submitted.  sync: the caller's thread also waits for the previous mutation; else
// its count is taken only if it has finished.
static int txid_begin(fabgpu_ctx* ctx, bool sync)
{
    auto& s = ctx->txid;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    if (!s.stream) {
        cudaStream_t st = nullptr; cudaEvent_t ev = nullptr;
        CK(ctx, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); s.stream.reset(st);
        CK(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); s.ev.reset(ev);
        for (auto& e : s.stage_ev) { cudaEvent_t x = nullptr; CK(ctx, cudaEventCreateWithFlags(&x, cudaEventDisableTiming)); e.reset(x); }
        if (int rc = s.d_count.reserve(ctx, 8)) return rc;
        if (int rc = s.h_count.reserve(ctx, 8)) return rc;
    }
    if (s.ev_set) {
        if (sync) CK(ctx, cudaEventSynchronize(s.ev.get()));
        const cudaError_t q = sync ? cudaSuccess : cudaEventQuery(s.ev.get());
        if (q == cudaSuccess) { s.count = s.h_count.get()[0]; s.pending = 0; }
        else if (q == cudaErrorNotReady) { if (cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError(); }
        else CK(ctx, q);
    }
    for (int k = 0; k < FABGPU_SLOTS; k++)
        if (s.decide_set[k]) CK(ctx, cudaStreamWaitEvent(s.stream.get(), s.decide_ev[k].get(), 0));
    return FABGPU_OK;
}

static uint64_t txid_max_bytes()
{
    const char* v = getenv("FABGPU_TXID_MAX_BYTES");      // bound on the table's bytes; unset = whatever cudaMalloc grants
    return v && *v ? strtoull(v, nullptr, 10) : ~0ull;
}

// Frees the table in stream order: the blocks that read it have been waited for (txid_begin)
static void txid_drop_table(fabgpu_ctx* ctx)
{
    auto& s = ctx->txid;
    if (s.table) cudaFreeAsync(s.table, s.stream.get());
    s.table = nullptr; s.slots = 0;
}

// Grows the table (doubling, to at least min_slots) so that `n` more ids fit at a load of at most 1/2
static int txid_room(fabgpu_ctx* ctx, uint64_t n, uint64_t min_slots)
{
    auto& s = ctx->txid;
    cudaStream_t st = s.stream.get();
    const uint64_t want = std::max(txid::slots_for(s.count + s.pending + n, s.slots), min_slots);
    if (want != s.slots) {
        const uint64_t bytes = want * sizeof(bdev::TxidSlot);
        if (bytes > txid_max_bytes() || want > (1ull << 32)) {
            char buf[192];
            snprintf(buf, sizeof buf, "committed tx-id table of %llu slots (%llu bytes) exceeds FABGPU_TXID_MAX_BYTES", (unsigned long long)want,
                     (unsigned long long)bytes);
            ctx->last_error = buf;
            return FABGPU_E_CUDA;
        }
        bdev::TxidSlot* nt = nullptr;
        CK(ctx, cudaMallocAsync(reinterpret_cast<void**>(&nt), bytes, st));
        if (cudaMemsetAsync(nt, 0, bytes, st) != cudaSuccess) { cudaFreeAsync(nt, st); ctx->last_error = "committed tx-id table clear failed"; return FABGPU_E_CUDA; }
        if (s.table) {
            bdev::txid_rehash_kernel<<<(unsigned)((s.slots + 255) / 256), 256, 0, st>>>(nt, (uint32_t)(want - 1), s.seed, s.table, s.slots);
            ctx->launches++;
            if (cudaGetLastError() != cudaSuccess) { cudaFreeAsync(nt, st); ctx->last_error = "committed tx-id rehash launch failed"; return FABGPU_E_CUDA; }
        }
        txid_drop_table(ctx);
        s.table = nt; s.slots = want;
    }
    return FABGPU_OK;
}

// Records the set event after the count's copy: later submits wait for it, and the next call takes the count once it has passed
static int txid_publish(fabgpu_ctx* ctx)
{
    auto& s = ctx->txid;
    cudaStream_t st = s.stream.get();
    CK(ctx, cudaMemcpyAsync(s.h_count.get(), s.d_count.get(), 8, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaEventRecord(s.ev.get(), st));
    s.ev_set = true;
    return FABGPU_OK;
}

// Grows the table so that `recs` fit, inserts them, and records the set event
static int txid_insert_records(fabgpu_ctx* ctx, const std::vector<bdev::TxidSlot>& recs, uint64_t min_slots)
{
    auto& s = ctx->txid;
    cudaStream_t st = s.stream.get();
    if (int rc = txid_room(ctx, recs.size(), min_slots)) return rc;
    const size_t n = recs.size();
    if (n) {
        const int r = (int)(s.seq++ % fabgpu_ctx::TxidSet::RING);
        auto& hs = s.h_stage[r];
        if (s.stage_set[r]) CK(ctx, cudaEventSynchronize(s.stage_ev[r].get()));     // its copy, RING mutations ago
        const size_t bytes = n * sizeof(bdev::TxidSlot);
        if (bytes > hs.bytes())
            if (int rc = hs.reserve(ctx, std::max(bytes, 2 * hs.bytes()))) return rc;
        if (bytes > s.d_stage.bytes())
            if (int rc = s.d_stage.reserve(ctx, std::max(bytes, 2 * s.d_stage.bytes()))) return rc;
        memcpy(hs.get(), recs.data(), bytes);
        CK(ctx, cudaMemcpyAsync(s.d_stage.get(), hs.get(), bytes, cudaMemcpyHostToDevice, st));
        CK(ctx, cudaEventRecord(s.stage_ev[r].get(), st));
        s.stage_set[r] = true;
        s.pending += n;
        bdev::txid_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.table, (uint32_t)(s.slots - 1), s.seed, s.d_stage.get(), (uint32_t)n,
                                                                             s.d_count.get());
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    return txid_publish(ctx);
}

// A failed mutation may have lost ids: from here on every lookup answers "unanswerable" (254) until a replacing call succeeds
static int txid_fail(fabgpu_ctx* ctx, int rc)
{
    auto& s = ctx->txid;
    const std::string err = ctx->last_error;
    s.broken = true;
    if (s.stream) {
        txid_drop_table(ctx);
        if (cudaEventRecord(s.ev.get(), s.stream.get()) == cudaSuccess) s.ev_set = true;
    }
    ctx->last_error = err + " (the committed tx-id set is broken until fabgpu_committed_txids replaces it)";
    return rc;
}

int fabgpu_committed_txids(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* kind, size_t n, size_t capacity_hint)
{
    if (!ctx) return FABGPU_E_ARG;
    std::vector<bdev::TxidSlot> recs;
    if (const char* err = txid::prepare(id_blob, id_off, kind, n, ctx->txid.seed, recs)) { ctx->last_error = err; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->txid;
    int rc = drain_block_streams(ctx);                         // a replacement is rare: it simply lets the blocks in flight finish
    if (!rc) rc = txid_begin(ctx, true);
    if (rc) return s.installed ? txid_fail(ctx, rc) : rc;
    txid_drop_table(ctx);
    s.installed = s.broken = false; s.count = s.pending = 0;
    if (n == 0 && capacity_hint == 0) {                        // removed: every flag is what it is without a set
        CK(ctx, cudaEventRecord(s.ev.get(), s.stream.get()));
        s.ev_set = true;
        return FABGPU_OK;
    }
    s.installed = true;
    CK(ctx, cudaMemsetAsync(s.d_count.get(), 0, 8, s.stream.get()));
    // the hint sizes the table up front when it fits under the byte bound; the ids given must fit in any case
    uint64_t hint_slots = txid::slots_for(capacity_hint);
    if (hint_slots * sizeof(bdev::TxidSlot) > txid_max_bytes()) hint_slots = 0;
    if ((rc = txid_insert_records(ctx, recs, hint_slots))) return txid_fail(ctx, rc);
    return FABGPU_OK;
}

int fabgpu_committed_txids_add(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* kind, size_t n)
{
    if (!ctx) return FABGPU_E_ARG;
    std::vector<bdev::TxidSlot> recs;
    if (const char* err = txid::prepare(id_blob, id_off, kind, n, ctx->txid.seed, recs)) { ctx->last_error = err; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->txid;
    if (!s.installed) { ctx->last_error = "no committed tx-id set installed: call fabgpu_committed_txids first"; return FABGPU_E_ARG; }
    if (s.broken) { ctx->last_error = "the committed tx-id set is broken by a failed call: replace it with fabgpu_committed_txids"; return FABGPU_E_ARG; }
    int rc = txid_begin(ctx, false);
    if (!rc) rc = txid_insert_records(ctx, recs, 0);
    return rc ? txid_fail(ctx, rc) : FABGPU_OK;
}

// The slot's block, on the set's stream after every slot's last decide stage (txid_begin): growth for T more ids, then
// txid_block_id_kernel (reads the slot's block and envelope table; read_ev follows it) and txid_block_insert_kernel (txidblock.cuh)
static int txid_insert_block(fabgpu_ctx* ctx, int slot)
{
    auto& s = ctx->txid; auto& db = ctx->dbs[slot];
    cudaStream_t st = s.stream.get();
    const uint32_t T = (uint32_t)db.T;
    if (int rc = txid_room(ctx, T, 0)) return rc;
    uint32_t dd = 64;
    while (dd < 2 * (uint64_t)T) dd <<= 1;
    Grow grow{ctx};
    grow(s.d_brec, sizeof(bdev::TxidSlot) * (size_t)T); grow(s.d_dd, 4 * (size_t)dd);
    if (grow.rc) return grow.rc;
    if (!s.read_ev[slot]) { cudaEvent_t ev = nullptr; CK(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); s.read_ev[slot].reset(ev); }
    CK(ctx, cudaMemsetAsync(s.d_dd.get(), 0, 4 * (size_t)dd, st));
    bdev::txid_block_id_kernel<<<(T + 127) / 128, 128, 0, st>>>(ctx->bbs[slot].d_block.get(), db.d_env_off.get(), T, s.d_brec.get());
    CK(ctx, cudaEventRecord(s.read_ev[slot].get(), st));
    s.read_set[slot] = true;
    bdev::txid_block_insert_kernel<<<(T + 255) / 256, 256, 0, st>>>(s.table, (uint32_t)(s.slots - 1), s.seed, s.d_brec.get(), T, s.d_dd.get(), dd - 1,
                                                                    s.d_count.get());
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    s.pending += T;
    return txid_publish(ctx);
}

int fabgpu_committed_txids_add_block(fabgpu_ctx* ctx, int slot)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->txid; auto& db = ctx->dbs[slot];
    if (!s.installed) { ctx->last_error = "no committed tx-id set installed: call fabgpu_committed_txids first"; return FABGPU_E_ARG; }
    if (s.broken) { ctx->last_error = "the committed tx-id set is broken by a failed call: replace it with fabgpu_committed_txids"; return FABGPU_E_ARG; }
    if (db.txid_block == 0) { ctx->last_error = "the slot holds no submitted block"; return FABGPU_E_ARG; }
    if (db.txid_block == 2) { ctx->last_error = "the slot's block was already added"; return FABGPU_E_ARG; }
    db.txid_block = 2;
    if (db.T == 0) return FABGPU_OK;
    int rc = txid_begin(ctx, false);
    if (!rc) rc = txid_insert_block(ctx, slot);
    return rc ? txid_fail(ctx, rc) : FABGPU_OK;
}

int fabgpu_committed_txids_info(const fabgpu_ctx* cctx, unsigned long long out[2])
{
    if (!cctx || !out) return FABGPU_E_ARG;
    fabgpu_ctx* ctx = const_cast<fabgpu_ctx*>(cctx);          // waits for the last mutation to read its count; changes nothing
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->txid;
    if (s.ev_set) {
        CK(ctx, cudaSetDevice(ctx->devs[0].id));
        CK(ctx, cudaEventSynchronize(s.ev.get()));
        if (s.installed && !s.broken) { s.count = s.h_count.get()[0]; s.pending = 0; }
    }
    out[0] = s.installed && !s.broken ? s.count : 0;
    out[1] = s.slots;
    return FABGPU_OK;
}

// ---- world-state version table and the MVCC stage (fabgpu_state_versions / _update / _info, fabgpu_validate_mvcc); under slot0_mu ----
static int sv_begin(fabgpu_ctx* ctx)
{
    auto& s = ctx->sv;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    if (!s.stream) {
        cudaStream_t st = nullptr;
        CK(ctx, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); s.stream.reset(st);
        if (int rc = s.d_count.reserve(ctx, 32)) return rc;
        if (int rc = s.h_count.reserve(ctx, 32)) return rc;
        if (int rc = s.d_ctr.reserve(ctx, 32)) return rc;
        if (int rc = s.h_ctr.reserve(ctx, 32)) return rc;
        if (int rc = s.d_icnt.reserve(ctx, 64)) return rc;
        if (int rc = s.h_icnt.reserve(ctx, 64)) return rc;
    }
    return FABGPU_OK;
}

static uint64_t sv_max_bytes()
{
    const char* v = getenv("FABGPU_STATE_MAX_BYTES");     // bound on the table's bytes; unset = whatever cudaMalloc grants
    return v && *v ? strtoull(v, nullptr, 10) : ~0ull;
}

// Bytes the index holds on the device (they count toward FABGPU_STATE_MAX_BYTES with the table's)
static uint64_t ix_bytes(fabgpu_ctx* ctx)
{
    auto& s = ctx->sv;
    return s.ix_base.bytes() + s.ix_delta.bytes() + s.ix_delta2.bytes() + s.ix_fresh.bytes() + s.ix_heap.bytes() + s.ix_flag.bytes();
}

static void ix_drop(fabgpu_ctx* ctx)
{
    auto& s = ctx->sv;
    s.indexed = false;
    s.ix_base = {}; s.ix_delta = {}; s.ix_delta2 = {}; s.ix_fresh = {}; s.ix_heap = {}; s.ix_flag = {};
    for (auto& c : s.icnt) c = 0;
}

static bdev::StateIndexDev ix_dev(fabgpu_ctx* ctx)
{
    auto& s = ctx->sv;
    bdev::StateIndexDev d{s.ix_base.get(), s.ix_delta.get(), s.ix_heap.get(), s.icnt[0], s.icnt[1], s.indexed ? 1u : 0u};
    return d;
}

static bdev::StateSetDev sv_dev(fabgpu_ctx* ctx)
{
    auto& s = ctx->sv;
    bdev::StateSetDev d{s.table, (uint32_t)(s.slots - 1), s.broken ? 1u : 0u, s.seed, s.d_count.get()};
    return d;
}

// Makes room for `more` further claimed slots at a load of at most 1/2 (and at least min_slots): a rehash into a fresh table on `st`,
// which drops removed keys.  The old table is freed in stream order.
static int sv_reserve(fabgpu_ctx* ctx, uint64_t more, uint64_t min_slots, cudaStream_t st)
{
    auto& s = ctx->sv;
    if (s.table && s.slots >= min_slots && s.count[1] + more <= s.slots / 2) return FABGPU_OK;
    const uint64_t want = std::max(stateset::slots_for(s.count[0] + more, s.slots), min_slots);
    const uint64_t bytes = want * sizeof(bdev::StateSlot);
    if (bytes + ix_bytes(ctx) > sv_max_bytes() || want > (1ull << 32)) {
        char buf[192];
        snprintf(buf, sizeof buf, "state version table of %llu slots (%llu bytes) exceeds FABGPU_STATE_MAX_BYTES", (unsigned long long)want,
                 (unsigned long long)bytes);
        ctx->last_error = buf;
        return FABGPU_E_CUDA;
    }
    bdev::StateSlot* nt = nullptr;
    CK(ctx, cudaMallocAsync(reinterpret_cast<void**>(&nt), bytes, st));
    if (cudaMemsetAsync(nt, 0, bytes, st) != cudaSuccess || cudaMemsetAsync(s.d_count.get(), 0, 24, st) != cudaSuccess) {
        cudaFreeAsync(nt, st); ctx->last_error = "state version table clear failed"; return FABGPU_E_CUDA;
    }
    bdev::StateSlot* old = s.table; const uint64_t n_old = s.slots;
    s.table = nt; s.slots = want;
    if (old) {
        bdev::sv_rehash_kernel<<<(unsigned)((n_old + 255) / 256), 256, 0, st>>>(sv_dev(ctx), old, n_old, reinterpret_cast<int*>(s.d_count.get() + 3));
        ctx->launches++;
        const cudaError_t e = cudaGetLastError();
        cudaFreeAsync(old, st);
        if (e != cudaSuccess) { ctx->last_error = "state version rehash launch failed"; return FABGPU_E_CUDA; }
    }
    s.count[1] = s.count[0];
    return FABGPU_OK;
}

// Upserts `recs` on `st` (room already made)
static int sv_insert(fabgpu_ctx* ctx, const std::vector<bdev::StateSlot>& recs, cudaStream_t st)
{
    auto& s = ctx->sv;
    const size_t n = recs.size();
    if (!n) return FABGPU_OK;
    const size_t bytes = n * sizeof(bdev::StateSlot);
    if (bytes > s.h_stage.bytes())
        if (int rc = s.h_stage.reserve(ctx, std::max(bytes, 2 * s.h_stage.bytes()))) return rc;
    if (bytes > s.d_stage.bytes())
        if (int rc = s.d_stage.reserve(ctx, std::max(bytes, 2 * s.d_stage.bytes()))) return rc;
    memcpy(s.h_stage.get(), recs.data(), bytes);
    CK(ctx, cudaMemcpyAsync(s.d_stage.get(), s.h_stage.get(), bytes, cudaMemcpyHostToDevice, st));
    bdev::sv_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(sv_dev(ctx), s.d_stage.get(), (uint32_t)n, reinterpret_cast<int*>(s.d_count.get() + 3));
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    return FABGPU_OK;
}

// Waits for `st` and takes the table's counts; a failed upsert (no free slot) is an error
static int sv_finish(fabgpu_ctx* ctx, cudaStream_t st)
{
    auto& s = ctx->sv;
    CK(ctx, cudaMemcpyAsync(s.h_count.get(), s.d_count.get(), 32, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < 3; k++) s.count[k] = s.h_count.get()[k];
    if (*reinterpret_cast<const int*>(s.h_count.get() + 3)) { ctx->last_error = "state version table: no free slot"; return FABGPU_E_CUDA; }
    return FABGPU_OK;
}

// FABGPU_OK, or the error text of a failed CUDA call that may have left the table half changed (the caller then breaks it, sv_fail)
static int sv_cuda(fabgpu_ctx* ctx, cudaError_t e, const char* what)
{
    if (e == cudaSuccess) return FABGPU_OK;
    ctx->last_error = std::string(what) + " failed: " + cudaGetErrorString(e);
    return FABGPU_E_CUDA;
}

// A failed call may have lost versions: every VALID transaction is 254 and nothing is applied until a replacing call succeeds
static int sv_fail(fabgpu_ctx* ctx, int rc, cudaStream_t st)
{
    auto& s = ctx->sv;
    const std::string err = ctx->last_error;
    s.broken = true;
    if (st) cudaStreamSynchronize(st);
    if (s.table) cudaFree(s.table);
    s.table = nullptr; s.slots = 0; s.count[0] = s.count[1] = s.count[2] = 0;
    ix_drop(ctx);
    ctx->last_error = err + " (the state version table is broken until fabgpu_state_versions replaces it)";
    return rc;
}

// Makes room in the index for a step adding at most `n_new` entries with at most `bytes_new` key bytes: the new run, its flags, the delta's
// next form (the merge writes it, then it becomes the delta), and the heap (grown with its contents kept)
static int ix_room(fabgpu_ctx* ctx, uint64_t n_new, uint64_t bytes_new, cudaStream_t st)
{
    auto& s = ctx->sv;
    const uint64_t E = sizeof(bdev::IndexEntry);
    const uint64_t want_fresh = std::max<uint64_t>(n_new, 1) * E, want_delta = (s.icnt[1] + std::max<uint64_t>(n_new, 1)) * E;
    const uint64_t want_heap = s.icnt[3] + bytes_new;
    uint64_t grow = 0;
    if (want_fresh > s.ix_fresh.bytes()) grow += 2 * want_fresh - s.ix_fresh.bytes();
    if (want_fresh / E * 4 > s.ix_flag.bytes()) grow += 2 * (want_fresh / E * 4);
    if (want_delta > s.ix_delta2.bytes()) grow += 2 * want_delta - s.ix_delta2.bytes();
    if (want_heap > s.ix_heap.bytes()) grow += 2 * want_heap;
    if (s.slots * sizeof(bdev::StateSlot) + ix_bytes(ctx) + grow > sv_max_bytes()) {
        ctx->last_error = "state key index exceeds FABGPU_STATE_MAX_BYTES";
        return FABGPU_E_CUDA;
    }
    Grow g{ctx};
    if (want_fresh > s.ix_fresh.bytes()) g(s.ix_fresh, 2 * want_fresh);
    if (want_fresh / E * 4 > s.ix_flag.bytes()) g(s.ix_flag, 2 * (want_fresh / E * 4));
    if (want_delta > s.ix_delta2.bytes()) g(s.ix_delta2, 2 * want_delta);
    if (g.rc) return g.rc;
    if (want_heap > s.ix_heap.bytes()) {
        DevArray<uint8_t> h;
        if (int rc = h.reserve(ctx, std::max<uint64_t>(2 * want_heap, 4096))) return rc;
        if (s.icnt[3]) CK(ctx, cudaMemcpyAsync(h.get(), s.ix_heap.get(), s.icnt[3], cudaMemcpyDeviceToDevice, st));
        CK(ctx, cudaStreamSynchronize(st));
        std::swap(h, s.ix_heap);
    }
    return FABGPU_OK;
}

// Adds to the index the candidates (sorted, at most n_ub of them, n_p: their device count, or n) that the table now holds and the
// index lacks: flags, the new run, its merge with the delta.  Room already made.  The counts are settled by ix_finish.
static int ix_insert(fabgpu_ctx* ctx, const bdev::WrittenKey* cand, uint32_t n, const uint32_t* n_p, uint64_t n_ub, const uint8_t* src, cudaStream_t st)
{
    auto& s = ctx->sv;
    if (!n_ub) return FABGPU_OK;
    const unsigned g1 = (unsigned)((n_ub + 255) / 256);
    bdev::ix_flag_kernel<<<g1, 256, 0, st>>>(cand, n, n_p, src, ix_dev(ctx), sv_dev(ctx), s.ix_flag.get());
    bdev::ix_compact_kernel<<<1, 1024, 0, st>>>(cand, n, n_p, src, s.ix_flag.get(), s.ix_heap.get(), s.ix_fresh.get(), s.d_icnt.get());
    bdev::ix_merge_kernel<<<(unsigned)((s.icnt[1] + n_ub + 255) / 256), 256, 0, st>>>(s.ix_delta.get(), s.d_icnt.get() + 1, s.ix_fresh.get(),
                                                                                     s.d_icnt.get() + 2, s.ix_heap.get(), s.ix_delta2.get());
    bdev::ix_fin_kernel<<<1, 1, 0, st>>>(s.d_icnt.get(), 0);
    ctx->launches += 4;
    CK(ctx, cudaGetLastError());
    std::swap(s.ix_delta, s.ix_delta2);
    return FABGPU_OK;
}

// Waits for `st`, takes the index's counts, and folds the delta into the base once it passes stateset::index_fold_at
static int ix_finish(fabgpu_ctx* ctx, cudaStream_t st)
{
    auto& s = ctx->sv;
    CK(ctx, cudaMemcpyAsync(s.h_icnt.get(), s.d_icnt.get(), 40, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < 5; k++) s.icnt[k] = s.h_icnt.get()[k];
    if (s.icnt[1] <= stateset::index_fold_at(s.icnt[0])) return FABGPU_OK;
    const uint64_t n = s.icnt[0] + s.icnt[1], E = sizeof(bdev::IndexEntry);
    if (s.slots * sizeof(bdev::StateSlot) + ix_bytes(ctx) + n * E > sv_max_bytes()) {
        ctx->last_error = "state key index exceeds FABGPU_STATE_MAX_BYTES";
        return FABGPU_E_CUDA;
    }
    DevArray<bdev::IndexEntry> nb;
    if (int rc = nb.reserve(ctx, n * E)) return rc;
    bdev::ix_merge_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.ix_base.get(), s.d_icnt.get(), s.ix_delta.get(), s.d_icnt.get() + 1,
                                                                      s.ix_heap.get(), nb.get());
    bdev::ix_fin_kernel<<<1, 1, 0, st>>>(s.d_icnt.get(), 1);
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaStreamSynchronize(st));
    std::swap(nb, s.ix_base);
    s.icnt[0] = n; s.icnt[1] = 0;
    return FABGPU_OK;
}

// Installs the index over the call's public keys (sorted on the host), on `st`
static int ix_install(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint32_t* coll_off, const uint8_t* key_blob,
                      const uint32_t* key_off, const uint64_t* ver, size_t n, const std::vector<bdev::StateSlot>& recs, cudaStream_t st)
{
    auto& s = ctx->sv;
    std::vector<bdev::WrittenKey> keys; std::vector<uint8_t> blob;
    stateset::index_keys(ns_blob, ns_off, coll_off, key_blob, key_off, ver, n, recs, keys, blob);
    std::vector<bdev::IndexEntry> ent(keys.size());
    for (size_t i = 0; i < keys.size(); i++) {
        ent[i].off = keys[i].ns_off; ent[i].nl = keys[i].nl; ent[i].kl = keys[i].kl;
        for (int k = 0; k < 8; k++) ent[i].w[k] = keys[i].w[k];
    }
    const uint64_t E = sizeof(bdev::IndexEntry), eb = std::max<uint64_t>(ent.size(), 1) * E, hb = std::max<uint64_t>(blob.size(), 4096);
    if (s.slots * sizeof(bdev::StateSlot) + eb + hb > sv_max_bytes()) { ctx->last_error = "state key index exceeds FABGPU_STATE_MAX_BYTES"; return FABGPU_E_CUDA; }
    Grow g{ctx};
    g(s.ix_base, eb); g(s.ix_heap, hb);
    if (g.rc) return g.rc;
    if (!ent.empty()) CK(ctx, cudaMemcpyAsync(s.ix_base.get(), ent.data(), ent.size() * E, cudaMemcpyHostToDevice, st));
    if (!blob.empty()) CK(ctx, cudaMemcpyAsync(s.ix_heap.get(), blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    unsigned long long* hc = s.h_icnt.get();
    hc[0] = ent.size(); hc[1] = 0; hc[2] = 0; hc[3] = blob.size(); hc[4] = 0;
    CK(ctx, cudaMemcpyAsync(s.d_icnt.get(), hc, 40, cudaMemcpyHostToDevice, st));
    s.indexed = true;
    return ix_finish(ctx, st);
}

// CouchDB: every public key the call gives a version is one CouchDB can hold (validateKey); false with the error text otherwise.  A
// removal passes: the stage marks unknown the keys a 254 transaction writes, such a key among them, and the caller settles it by removal.
static bool cv_keys_ok(fabgpu_ctx* ctx, const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n)
{
    for (size_t i = 0; i < n; i++)
        if (coll_off[i + 1] == coll_off[i] && !(ver[2 * i] == UINT64_MAX && ver[2 * i + 1] == UINT64_MAX) &&
            !bdev::cv_key_ok(key_blob + key_off[i], key_off[i + 1] - key_off[i])) {
            ctx->last_error = "a public key CouchDB cannot hold (empty, starting with '_', or not UTF-8) under FABGPU_STATEDB_COUCHDB";
            return false;
        }
    return true;
}

static int sv_replace(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                      const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height, size_t capacity_hint, bool indexed)
{
    if (!ctx) return FABGPU_E_ARG;
    std::vector<bdev::StateSlot> recs;
    if (const char* err = stateset::prepare(ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, ver, n, ctx->sv.seed, recs)) { ctx->last_error = err; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    s.upd_slot = -1;
    if (s.couch && !cv_keys_ok(ctx, coll_off, key_blob, key_off, ver, n)) return FABGPU_E_ARG;
    int rc = drain_block_streams(ctx);                         // the stage of a slot's block may still be running: let it finish
    if (!rc) rc = sv_begin(ctx);
    if (rc) return s.installed ? sv_fail(ctx, rc, nullptr) : rc;
    cudaStream_t st = s.stream.get();
    if (s.table) cudaFreeAsync(s.table, st);
    s.table = nullptr; s.slots = 0; s.count[0] = s.count[1] = s.count[2] = 0;
    s.installed = s.broken = s.open = false; s.height = 0;
    if (s.indexed) { CK(ctx, cudaStreamSynchronize(st)); ix_drop(ctx); }
    if (n == 0 && capacity_hint == 0) { CK(ctx, cudaStreamSynchronize(st)); return FABGPU_OK; }
    s.installed = true; s.height = height;
    uint64_t hint_slots = stateset::slots_for(capacity_hint);
    if (hint_slots * sizeof(bdev::StateSlot) > sv_max_bytes()) hint_slots = 0;
    if ((rc = sv_cuda(ctx, cudaMemsetAsync(s.d_count.get(), 0, 32, st), "state version count clear")) ||
        (rc = sv_reserve(ctx, recs.size(), hint_slots, st)) || (rc = sv_insert(ctx, recs, st)) || (rc = sv_finish(ctx, st)) ||
        (indexed && (rc = ix_install(ctx, ns_blob, ns_off, coll_off, key_blob, key_off, ver, n, recs, st))))
        return sv_fail(ctx, rc, st);
    return FABGPU_OK;
}

int fabgpu_state_versions(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                          const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height, size_t capacity_hint)
{
    return sv_replace(ctx, ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, ver, n, height, capacity_hint, false);
}

int fabgpu_state_versions_indexed(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                                  const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height, size_t capacity_hint)
{
    return sv_replace(ctx, ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, ver, n, height, capacity_hint, true);
}

int fabgpu_state_versions_update(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                                 const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height)
{
    if (!ctx) return FABGPU_E_ARG;
    std::vector<bdev::StateSlot> recs;
    if (const char* err = stateset::prepare(ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, ver, n, ctx->sv.seed, recs)) { ctx->last_error = err; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    s.upd_slot = -1;
    if (!s.installed) { ctx->last_error = "no state version table installed: call fabgpu_state_versions first"; return FABGPU_E_ARG; }
    if (s.broken) { ctx->last_error = "the state version table is broken by a failed call: replace it with fabgpu_state_versions"; return FABGPU_E_ARG; }
    if (s.couch && !cv_keys_ok(ctx, coll_off, key_blob, key_off, ver, n)) return FABGPU_E_ARG;
    if (height < s.height) { ctx->last_error = "state version height below the table's height"; return FABGPU_E_ARG; }
    int rc = sv_begin(ctx);
    if (rc) return rc;
    cudaStream_t st = s.stream.get();
    if ((rc = sv_reserve(ctx, recs.size(), 0, st)) || (rc = sv_insert(ctx, recs, st)) || (rc = sv_finish(ctx, st))) return sv_fail(ctx, rc, st);
    if (s.indexed) {                                           // the index gains the public keys it lacks
        std::vector<bdev::WrittenKey> keys; std::vector<uint8_t> blob;
        stateset::index_keys(ns_blob, ns_off, coll_off, key_blob, key_off, ver, n, recs, keys, blob);
        if (!keys.empty()) {
            Grow g{ctx};
            g(s.d_cand, keys.size() * sizeof(bdev::WrittenKey)); g(s.d_cand_bytes, std::max<size_t>(blob.size(), 1));
            if (g.rc) return sv_fail(ctx, g.rc, st);
            if ((rc = sv_cuda(ctx, cudaMemcpyAsync(s.d_cand.get(), keys.data(), keys.size() * sizeof(bdev::WrittenKey), cudaMemcpyHostToDevice, st), "index copy")) ||
                (!blob.empty() && (rc = sv_cuda(ctx, cudaMemcpyAsync(s.d_cand_bytes.get(), blob.data(), blob.size(), cudaMemcpyHostToDevice, st), "index copy"))) ||
                (rc = ix_room(ctx, keys.size(), blob.size(), st)) ||
                (rc = ix_insert(ctx, s.d_cand.get(), (uint32_t)keys.size(), nullptr, keys.size(), s.d_cand_bytes.get(), st)) || (rc = ix_finish(ctx, st)))
                return sv_fail(ctx, rc, st);
        }
    }
    if (height > s.height) { s.height = height; s.open = false; }
    return FABGPU_OK;
}

int fabgpu_state_index_info(const fabgpu_ctx* cctx, unsigned long long out[3])
{
    if (!cctx || !out) return FABGPU_E_ARG;
    fabgpu_ctx* ctx = const_cast<fabgpu_ctx*>(cctx);          // takes slot0_mu; changes nothing the stage reads
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    out[0] = out[1] = out[2] = 0;
    if (!s.indexed || !s.installed || s.broken) return FABGPU_OK;
    if (int rc = sv_begin(ctx)) return rc;
    cudaStream_t st = s.stream.get();
    const uint64_t n = s.icnt[0] + s.icnt[1];
    CK(ctx, cudaMemsetAsync(s.d_icnt.get() + 4, 0, 8, st));
    if (n) {
        bdev::ix_live_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ix_dev(ctx), sv_dev(ctx), s.d_icnt.get());
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    CK(ctx, cudaMemcpyAsync(s.h_icnt.get(), s.d_icnt.get(), 40, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    out[0] = s.h_icnt.get()[4]; out[1] = n; out[2] = ix_bytes(ctx);
    return FABGPU_OK;
}

int fabgpu_state_versions_info(const fabgpu_ctx* cctx, unsigned long long out[4])
{
    if (!cctx || !out) return FABGPU_E_ARG;
    fabgpu_ctx* ctx = const_cast<fabgpu_ctx*>(cctx);          // takes slot0_mu; changes nothing
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    const bool on = s.installed && !s.broken;
    out[0] = on ? s.count[0] : 0; out[1] = s.slots; out[2] = s.height; out[3] = on ? s.count[2] : 0;
    return FABGPU_OK;
}

int fabgpu_state_database(fabgpu_ctx* ctx, int kind)
{
    if (!ctx) return FABGPU_E_ARG;
    if (kind != FABGPU_STATEDB_LEVELDB && kind != FABGPU_STATEDB_COUCHDB) { ctx->last_error = "unknown state database kind"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    ctx->sv.couch = kind == FABGPU_STATEDB_COUCHDB;
    return FABGPU_OK;
}

// CouchDB's pre-pass on `st`, before the stage reads d_tv: cv_scan_kernel (per transaction: the public writes of the VALID ones, and
// the read / range rules) -> host reads the write count (grows the arrays and runs the scan again on overflow) -> cv_check_kernel (per
// write: key, and a value of at most CV_SHORT_MAX bytes) -> cv_long_kernel (one CTA per longer value) -> cv_flag_kernel (per transaction: VALID -> 24 or 254 in d_tv)
static int cv_prepass(fabgpu_ctx* ctx, cudaStream_t st, const uint8_t* blk, const bdev::TxDev* txs, uint32_t T)
{
    auto& s = ctx->sv;
    Grow grow{ctx};
    grow(s.d_cv_first, 4 * (size_t)T); grow(s.d_cv_n, 4 * (size_t)T); grow(s.d_cv_undet, T);
    if (grow.rc) return grow.rc;
    bdev::CvArrays c;
    uint32_t W = 0;
    for (;;) {
        const size_t W_cap = (size_t)T * s.cv_hint;
        if (W_cap > UINT32_MAX) { ctx->last_error = "block has too many writes"; return FABGPU_E_ARG; }
        Grow g2{ctx};
        g2(s.d_cvw, W_cap * sizeof(bdev::CvWrite)); g2(s.d_cv_code, W_cap); g2(s.d_cv_long, 4 * W_cap);
        if (g2.rc) return g2.rc;
        uint32_t* hc = s.h_ctr.get();
        hc[0] = hc[1] = 0;
        CK(ctx, cudaMemcpyAsync(s.d_ctr.get(), hc, 8, cudaMemcpyHostToDevice, st));
        c.w = s.d_cvw.get(); c.W_cap = (uint32_t)W_cap; c.first_w = s.d_cv_first.get(); c.n_w = s.d_cv_n.get(); c.undet = s.d_cv_undet.get();
        c.code = s.d_cv_code.get(); c.lng = s.d_cv_long.get(); c.ctr = s.d_ctr.get();
        bdev::cv_scan_kernel<<<(T + 63) / 64, 64, 0, st>>>(blk, txs, T, s.d_tv.get(), c);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(hc, s.d_ctr.get(), 4, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
        W = hc[0];
        if (W <= W_cap) break;
        s.cv_hint = (uint32_t)((W + T - 1) / T) + 1;
    }
    if (W) {                                                   // the long values: one CTA each, as many as there are (at most 264 CTAs)
        bdev::cv_check_kernel<<<(W + 127) / 128, 128, 0, st>>>(blk, c, W);
        bdev::cv_long_kernel<<<std::min(W, 264u), bdev::CV_LT_THREADS, 0, st>>>(blk, c);
        ctx->launches += 2;
    }
    bdev::cv_flag_kernel<<<(T + 127) / 128, 128, 0, st>>>(c, s.d_tv.get(), T);
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    return FABGPU_OK;
}

// The stage ran on the slot's block: fabgpu_block_updates may build its batch from the stage's arrays (R records, K key-table entries)
static void upd_mark(fabgpu_ctx* ctx, int slot, uint64_t block_num, uint32_t R, uint32_t K, uint32_t T, bool incomplete, const uint8_t* flags, size_t n)
{
    auto& s = ctx->sv;
    s.upd_flags.assign(flags, flags + n);
    s.upd_slot = slot; s.upd_block = block_num; s.upd_R = R; s.upd_K = K; s.upd_T = T;
    s.upd_incomplete = incomplete; s.upd_built = false; s.upd_ordered = false; s.upd_n[0] = s.upd_n[1] = 0;
    ctx->dbs[slot].upd_ready = true;
}

// The MVCC stage of the slot's block, on the slot's stream after its last kernel:
//   mv_scan_kernel (per transaction: read / write records with key digests) -> host reads the record count (grows the arrays and runs
//   the scan again on overflow) -> mv_key_kernel (per record: the block's key table, the committed table's answer) -> mv_check_kernel
//   -> mv_mark_kernel (per transaction: flags of the independent ones) -> mv_walk_kernel (one thread: the dependent ones in order)
//   -> growth of the table for the block's keys -> mv_apply_kernel (per key: its final state at (block_num, tx)) -> D2H flags.
// Under CouchDB, cv_prepass runs first and turns VALID flags of d_tv into 24 or 254, so a 24 transaction drops out of the stage.
// With an index installed the scan also emits range records, and before mv_mark_kernel: mv_written_kernel (the block's written public
// keys) -> mv_sort_kernel (one launch per merge pass) -> mv_range_kernel (per range record: marking and the committed answer); after the
// apply the index gains the block's new keys (ix_insert), and the delta is folded into the base when due (ix_finish).
int fabgpu_validate_mvcc(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* tv_flags, uint8_t* flags, size_t n)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (n && (!tv_flags || !flags)) { ctx->last_error = "flag arrays missing"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv; auto& db = ctx->dbs[slot];
    s.upd_slot = -1;
    if (!s.installed) { ctx->last_error = "no state version table installed: call fabgpu_state_versions first"; return FABGPU_E_ARG; }
    if (s.open) { ctx->last_error = "the previous block is open: fabgpu_state_versions_update(..., height = block_num + 1) first"; return FABGPU_E_ARG; }
    if (block_num != s.height) { ctx->last_error = "block_num is not the table's height"; return FABGPU_E_ARG; }
    if (db.busy || !db.mvcc_ready) { ctx->last_error = "the slot holds no finished block: fabgpu_validate_wait first"; return FABGPU_E_ARG; }
    if (n != db.T) { ctx->last_error = "n is not the block's transaction count"; return FABGPU_E_ARG; }
    if (s.broken) {                                            // nothing can be decided or applied
        for (size_t t = 0; t < n; t++) flags[t] = tv_flags[t] == bdev::TXC_VALID ? bdev::TXC_NOT_VALIDATED : tv_flags[t];
        upd_mark(ctx, slot, block_num, 0, 0, 0, true, flags, n);
        return FABGPU_OK;
    }
    int rc = sv_begin(ctx);
    if (rc) return rc;
    const uint32_t T = (uint32_t)n;
    if (T == 0) { db.mvcc_ready = false; s.height = block_num + 1; upd_mark(ctx, slot, block_num, 0, 0, 0, false, flags, 0); return FABGPU_OK; }
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    Grow grow{ctx};
    grow(s.d_first, 4 * (size_t)T); grow(s.d_n, 4 * (size_t)T); grow(s.d_mlist, 4 * (size_t)T); grow(s.d_info, T); grow(s.d_tv, T); grow(s.d_flags, T);
    grow(s.h_flags, T);
    if (grow.rc) return grow.rc;
    memcpy(s.h_flags.get(), tv_flags, n);
    CK(ctx, cudaMemcpyAsync(s.d_tv.get(), s.h_flags.get(), n, cudaMemcpyHostToDevice, st));
    const uint8_t* blk = ctx->bbs[slot].d_block.get();
    if (s.couch && (rc = cv_prepass(ctx, st, blk, db.d_txs.get(), T))) return rc;
    const bool ix = s.indexed;
    if (ix) {
        grow(s.d_first_rng, 4 * (size_t)T); grow(s.d_n_rng, 4 * (size_t)T);
        if (grow.rc) return grow.rc;
    }
    bdev::MvccArrays a;
    uint32_t R = 0, G = 0;
    for (;;) {
        const size_t R_cap = (size_t)T * s.rec_hint, G_cap = ix ? (size_t)T * s.rng_hint : 0;
        if (R_cap > UINT32_MAX || G_cap > UINT32_MAX) { ctx->last_error = "block has too many read and write records"; return FABGPU_E_ARG; }
        if (R_cap * sizeof(bdev::MvccRec) > s.d_rec.bytes())
            if (int r2 = s.d_rec.reserve(ctx, R_cap * sizeof(bdev::MvccRec))) return r2;
        if (G_cap * sizeof(bdev::MvccRange) > s.d_rng.bytes())
            if (int r2 = s.d_rng.reserve(ctx, G_cap * sizeof(bdev::MvccRange))) return r2;
        uint32_t* hc = s.h_ctr.get();
        hc[0] = 0; hc[1] = 0; hc[2] = UINT32_MAX; hc[3] = 0; hc[4] = 0; hc[5] = 0; hc[6] = 0; hc[7] = 0;
        CK(ctx, cudaMemcpyAsync(s.d_ctr.get(), hc, 32, cudaMemcpyHostToDevice, st));
        a.rec = s.d_rec.get(); a.R_cap = (uint32_t)R_cap; a.first_rec = s.d_first.get(); a.n_rec = s.d_n.get(); a.info = s.d_info.get();
        a.key = nullptr; a.K_size = 0; a.ctr = s.d_ctr.get(); a.mlist = s.d_mlist.get();
        if (ix) {
            a.indexed = 1; a.block = block_num; a.rng = s.d_rng.get(); a.G_cap = (uint32_t)G_cap; a.first_rng = s.d_first_rng.get();
            a.n_rng = s.d_n_rng.get(); a.ix = ix_dev(ctx);
        }
        bdev::mv_scan_kernel<<<(T + 63) / 64, 64, 0, st>>>(blk, db.d_txs.get(), T, s.d_tv.get(), a);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(hc, s.d_ctr.get(), 32, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
        R = hc[0]; G = hc[4];
        if (R <= R_cap && G <= G_cap) break;
        if (R > R_cap) s.rec_hint = (uint32_t)((R + T - 1) / T) + 1;            // later blocks are sized for it too
        if (G > G_cap) s.rng_hint = (uint32_t)((G + T - 1) / T) + 1;
    }
    const uint64_t key_bytes = s.h_ctr.get()[6];
    uint32_t K = 64;
    while (K < 2 * (uint64_t)R) K <<= 1;
    if ((size_t)K * sizeof(bdev::MvccKey) > s.d_key.bytes())
        if (int r2 = s.d_key.reserve(ctx, (size_t)K * sizeof(bdev::MvccKey))) return r2;
    a.key = s.d_key.get(); a.K_size = K;
    CK(ctx, cudaMemsetAsync(a.key, 0, (size_t)K * sizeof(bdev::MvccKey), st));
    if (R) {
        bdev::mv_key_kernel<<<(R + 255) / 256, 256, 0, st>>>(a, sv_dev(ctx), R);
        bdev::mv_check_kernel<<<(R + 255) / 256, 256, 0, st>>>(a, R);
        ctx->launches += 2;
    }
    if (ix && (R || G)) {                                      // the block's written public keys, sorted (at most R of them)
        Grow g2{ctx};
        g2(s.d_wk, (size_t)std::max(R, 1u) * sizeof(bdev::WrittenKey)); g2(s.d_wk2, (size_t)std::max(R, 1u) * sizeof(bdev::WrittenKey));
        if (g2.rc) return g2.rc;
        a.wk = s.d_wk.get();
        bdev::mv_written_kernel<<<(K + 255) / 256, 256, 0, st>>>(a);
        ctx->launches++;
        bdev::WrittenKey* in = s.d_wk.get(); bdev::WrittenKey* out = s.d_wk2.get();
        for (uint32_t width = 1; width < R; width <<= 1) {
            bdev::mv_sort_kernel<<<(R + 255) / 256, 256, 0, st>>>(in, out, a.ctr, width, blk);
            ctx->launches++;
            std::swap(in, out);
        }
        a.wk = in;
        if (G) {
            if ((size_t)G * sizeof(bdev::MerkleState) > s.d_mk.bytes())
                if (int r2 = s.d_mk.reserve(ctx, (size_t)G * sizeof(bdev::MerkleState))) return r2;
            a.mk = s.d_mk.get();
            bdev::mv_range_kernel<<<(G + 127) / 128, 128, 0, st>>>(blk, a, sv_dev(ctx), G);
            ctx->launches++;
        }
    }
    bdev::mv_mark_kernel<<<(T + 127) / 128, 128, 0, st>>>(s.d_tv.get(), a, s.d_flags.get(), T);
    if (ix) bdev::mv_walk_kernel<true><<<1, 256, 0, st>>>(s.d_tv.get(), a, s.d_flags.get(), T, blk, sv_dev(ctx));
    else bdev::mv_walk_kernel<false><<<1, 256, 0, st>>>(s.d_tv.get(), a, s.d_flags.get(), T, blk, sv_dev(ctx));
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    if ((rc = sv_reserve(ctx, R, 0, st))) return sv_fail(ctx, rc, st);
    if (ix && R && (rc = ix_room(ctx, R, key_bytes, st))) return sv_fail(ctx, rc, st);
    bdev::mv_apply_kernel<<<(K + 255) / 256, 256, 0, st>>>(a, s.d_flags.get(), sv_dev(ctx), (unsigned long long)block_num,
                                                          reinterpret_cast<int*>(s.d_count.get() + 3));
    ctx->launches++;
    // from the apply on the table is changed: a failure leaves it broken
    if (ix && R && (rc = ix_insert(ctx, a.wk, 0, a.ctr + 5, R, blk, st))) return sv_fail(ctx, rc, st);
    if ((rc = sv_cuda(ctx, cudaGetLastError(), "mv_apply_kernel launch")) ||
        (rc = sv_cuda(ctx, cudaMemcpyAsync(s.h_flags.get(), s.d_flags.get(), n, cudaMemcpyDeviceToHost, st), "MVCC flag copy")) ||
        (rc = sv_cuda(ctx, cudaMemcpyAsync(s.h_ctr.get(), s.d_ctr.get(), 16, cudaMemcpyDeviceToHost, st), "MVCC counter copy")) ||
        (rc = sv_finish(ctx, st)) || (ix && R && (rc = ix_finish(ctx, st))))
        return sv_fail(ctx, rc, st);
    memcpy(flags, s.h_flags.get(), n);
    const uint32_t* hc = s.h_ctr.get();
    db.mvcc_ready = false;
    if (hc[1] || hc[2] != UINT32_MAX) s.open = true;           // two keys shared a tag, or a write set could not be enumerated
    else s.height = block_num + 1;
    upd_mark(ctx, slot, block_num, R, K, T, s.open, flags, n);
    return FABGPU_OK;
}

// The private-data arrays' refusals that need no lock: decreasing offsets, a missing blob, sizes past 32 bits
static int pvt_args(fabgpu_ctx* ctx, const uint8_t* pvt_blob, const uint32_t* pvt_off, size_t n_pvt)
{
    for (size_t i = 0; i < n_pvt; i++) if (pvt_off[i + 1] < pvt_off[i]) { ctx->last_error = "private-data offsets decrease"; return FABGPU_E_ARG; }
    const size_t bytes = n_pvt ? pvt_off[n_pvt] : 0;
    if (bytes && !pvt_blob) { ctx->last_error = "arrays missing"; return FABGPU_E_ARG; }
    if (n_pvt > UINT32_MAX || bytes > UINT32_MAX - 64) { ctx->last_error = "too much private data for one call"; return FABGPU_E_ARG; }
    return FABGPU_OK;
}

// Every seq below the block's transaction count n, none given twice
static int pvt_seqs(fabgpu_ctx* ctx, const uint32_t* seq, size_t n_pvt, size_t n)
{
    std::vector<uint8_t> seen(n, 0);
    for (size_t i = 0; i < n_pvt; i++) {
        if (seq[i] >= n) { ctx->last_error = "a seq is not below the block's transaction count"; return FABGPU_E_ARG; }
        if (seen[seq[i]]++) { ctx->last_error = "a seq is given twice"; return FABGPU_E_ARG; }
    }
    return FABGPU_OK;
}

// The private-data check of the slot's block, on the slot's stream under blk_mu[slot] (arguments already checked; returns synchronised):
//   H2D private data, entry tables, flags -> pv_scan_kernel (per entry: collection records, SHA-256 jobs) -> host reads the record count
//   (grows the arrays and runs the scan again on overflow) -> sha256_segments_kernel (per record: its rwset) -> pv_check_kernel (per
//   record: the public hash, the decode) -> pv_verdict_kernel (per entry: its outcome, atomicMin of the deciding entry) -> D2H.
// The records, the flags and the private data stay on the device for fabgpu_block_pvt_updates; R_out: the record count.
static int pvt_check(fabgpu_ctx* ctx, int slot, const uint8_t* flags, size_t n, const uint8_t* pvt_blob, const uint32_t* pvt_off,
                     const uint32_t* seq, size_t n_pvt, int32_t* status, int32_t out[4], uint32_t& R_out)
{
    auto& db = ctx->dbs[slot]; auto& p = ctx->pvt[slot];
    R_out = 0;
    out[0] = bdev::PV_OK; out[1] = out[2] = out[3] = -1;
    if (n_pvt == 0) return FABGPU_OK;
    const size_t bytes = pvt_off[n_pvt];
    const uint32_t E = (uint32_t)n_pvt, T = (uint32_t)n;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    Grow grow{ctx};
    // slack: the SHA-256 loader reads the aligned words past a range's end
    grow(p.h_blob, bytes + 64); grow(p.h_flags, T); grow(p.h_off, 4 * ((size_t)E + 1)); grow(p.h_seq, 4 * (size_t)E); grow(p.h_ctr, 16);
    grow(p.h_status, 12 * (size_t)E); grow(p.h_verdict, 8);
    grow(p.d_blob, bytes + 64); grow(p.d_flags, T); grow(p.d_off, 4 * ((size_t)E + 1)); grow(p.d_seq, 4 * (size_t)E); grow(p.d_ent, E);
    grow(p.d_first, 4 * (size_t)E); grow(p.d_n, 4 * (size_t)E); grow(p.d_ctr, 16); grow(p.d_status, 12 * (size_t)E); grow(p.d_verdict, 8);
    if (grow.rc) return grow.rc;
    memcpy(p.h_blob.get(), pvt_blob, bytes); memset(p.h_blob.get() + bytes, 0, 64);
    memcpy(p.h_flags.get(), flags, n); memcpy(p.h_off.get(), pvt_off, 4 * ((size_t)E + 1)); memcpy(p.h_seq.get(), seq, 4 * (size_t)E);
    CK(ctx, cudaMemcpyAsync(p.d_blob.get(), p.h_blob.get(), bytes + 64, cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(p.d_flags.get(), p.h_flags.get(), n, cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(p.d_off.get(), p.h_off.get(), 4 * ((size_t)E + 1), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(p.d_seq.get(), p.h_seq.get(), 4 * (size_t)E, cudaMemcpyHostToDevice, st));
    const uint8_t* blk = ctx->bbs[slot].d_block.get();
    bdev::PvArrays a;
    a.pvt = p.d_blob.get(); a.off = p.d_off.get(); a.seq = p.d_seq.get(); a.n_pvt = E; a.flags = p.d_flags.get(); a.ent = p.d_ent.get();
    a.first = p.d_first.get(); a.n_rec = p.d_n.get(); a.ctr = p.d_ctr.get(); a.status = p.d_status.get(); a.verdict = p.d_verdict.get();
    uint32_t R = 0;
    for (;;) {
        const size_t R_cap = (size_t)E * p.rec_hint;
        if (R_cap > UINT32_MAX) { ctx->last_error = "too many collections for one call"; return FABGPU_E_ARG; }
        Grow g2{ctx};
        g2(p.d_rec, R_cap * sizeof(bdev::PvRec)); g2(p.d_jobs, R_cap * sizeof(bdev::ShaJobP)); g2(p.d_dig, 32 * R_cap);
        if (g2.rc) return g2.rc;
        a.rec = p.d_rec.get(); a.R_cap = (uint32_t)R_cap; a.jobs = p.d_jobs.get(); a.dig = p.d_dig.get();
        CK(ctx, cudaMemsetAsync(p.d_ctr.get(), 0, 16, st));
        bdev::pv_scan_kernel<<<(E + 63) / 64, 64, 0, st>>>(blk, db.d_txs.get(), a);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(p.h_ctr.get(), p.d_ctr.get(), 4, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
        R = p.h_ctr.get()[0];
        if (R <= R_cap) break;
        p.rec_hint = (uint32_t)((R + E - 1) / E) + 1;                   // later calls are sized for it too
    }
    if (R) {
        sha256_segments_kernel<<<(R + 127) / 128, 128, 0, st>>>(p.d_blob.get(), reinterpret_cast<const ShaJob*>(p.d_jobs.get()), R, p.d_dig.get());
        bdev::pv_check_kernel<<<(R + 127) / 128, 128, 0, st>>>(blk, db.d_txs.get(), a, R);
        ctx->launches += 2;
    }
    CK(ctx, cudaMemsetAsync(p.d_verdict.get(), 0xff, 8, st));
    bdev::pv_verdict_kernel<<<(E + 127) / 128, 128, 0, st>>>(a);
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(p.h_status.get(), p.d_status.get(), 12 * (size_t)E, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaMemcpyAsync(p.h_verdict.get(), p.d_verdict.get(), 8, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    memcpy(status, p.h_status.get(), 12 * (size_t)E);
    const unsigned long long v = p.h_verdict.get()[0];
    if (v != ~0ull) {                                          // the deciding entry: a mismatch when its flag is VALID, else 254
        const uint32_t e = (uint32_t)v, s = (uint32_t)(v >> 32);
        const int32_t* es = status + 3 * (size_t)e;
        const bool mismatch = es[0] == bdev::PV_MISMATCH && flags[s] == bdev::TXC_VALID;
        out[0] = mismatch ? bdev::PV_MISMATCH : bdev::PV_UNDET; out[1] = (int32_t)s;
        out[2] = mismatch ? es[1] : -1; out[3] = mismatch ? es[2] : -1;
    }
    R_out = R;
    return FABGPU_OK;
}

int fabgpu_validate_pvtdata(fabgpu_ctx* ctx, int slot, const uint8_t* flags, size_t n, const uint8_t* pvt_blob, const uint32_t* pvt_off,
                            const uint32_t* seq, size_t n_pvt, int32_t* status, int32_t out[4])
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || !out) return FABGPU_E_ARG;
    if ((n && !flags) || (n_pvt && (!pvt_off || !seq || !status))) { ctx->last_error = "arrays missing"; return FABGPU_E_ARG; }
    if (int rc = pvt_args(ctx, pvt_blob, pvt_off, n_pvt)) return rc;
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    auto& db = ctx->dbs[slot];
    if (db.busy || !db.pvt_ready) { ctx->last_error = "the slot holds no finished block: fabgpu_validate_wait first"; return FABGPU_E_ARG; }
    if (n != db.T) { ctx->last_error = "n is not the block's transaction count"; return FABGPU_E_ARG; }
    if (int rc = pvt_seqs(ctx, seq, n_pvt, n)) return rc;
    uint32_t R;
    return pvt_check(ctx, slot, flags, n, pvt_blob, pvt_off, seq, n_pvt, status, out, R);
}

int fabgpu_block_unknown_identities(fabgpu_ctx* ctx, int slot, uint32_t* out, size_t cap, size_t* n_out)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (!n_out || (cap && !out)) { ctx->last_error = "output arrays missing"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    auto& db = ctx->dbs[slot]; auto& u = ctx->uk[slot];
    if (db.busy || !db.pvt_ready) { ctx->last_error = "the slot holds no finished block: fabgpu_validate_wait first"; return FABGPU_E_ARG; }
    *n_out = 0;
    if (db.T == 0) return FABGPU_OK;
    const uint32_t T = (uint32_t)db.T, J = (uint32_t)(db.T * (1 + BD_ENDS_HINT));
    uint32_t slots = 16; while (slots < 2 * J) slots <<= 1;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    Grow grow{ctx};
    grow(u.d_hash, 8 * (size_t)J); grow(u.d_index, 4 * (size_t)slots); grow(u.d_rep, 4 * (size_t)J); grow(u.d_first, 8 * (size_t)J);
    grow(u.d_cnt, 4 * ((size_t)T + 1)); grow(u.d_out, 12 * (size_t)J); grow(u.h_cnt, 4); grow(u.h_out, 12 * (size_t)J);
    if (grow.rc) return grow.rc;
    bdev::UkArrays a;
    a.raw = db.d_raw.get(); a.ident = db.d_ident.get(); a.txs = db.d_txs.get(); a.T = T; a.E_cap = J - T; a.n_end = db.d_counter.get();
    a.hash = u.d_hash.get(); a.index = u.d_index.get(); a.index_mask = slots - 1; a.rep = u.d_rep.get(); a.first = u.d_first.get();
    a.cnt = u.d_cnt.get(); a.out = u.d_out.get();
    const uint8_t* blk = ctx->bbs[slot].d_block.get();
    CK(ctx, cudaMemsetAsync(u.d_index.get(), 0xff, 4 * (size_t)slots, st));
    bdev::uk_hash_kernel<<<(J + 127) / 128, 128, 0, st>>>(blk, a);
    bdev::uk_insert_kernel<<<(J + 127) / 128, 128, 0, st>>>(blk, a);
    bdev::uk_count_kernel<<<(T + 127) / 128, 128, 0, st>>>(a);
    bdev::uk_scan_kernel<<<1, 1024, 0, st>>>(a);
    bdev::uk_emit_kernel<<<(T + 127) / 128, 128, 0, st>>>(a);
    ctx->launches += 5;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(u.h_cnt.get(), u.d_cnt.get() + T, 4, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    const size_t total = u.h_cnt.get()[0], w = std::min(total, cap);
    if (w) {
        CK(ctx, cudaMemcpyAsync(u.h_out.get(), u.d_out.get(), 12 * w, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
        memcpy(out, u.h_out.get(), 12 * w);
    }
    *n_out = total;
    return FABGPU_OK;
}

// Builds the update batch of the block the stage last ran on (on `slot`'s stream; returns synchronised):
//   ud_pair_kernel (per record: (tx, key) pairs of VALID writes) -> ud_class_kernel (per pair) -> ud_walk_kernel (per pair: the nearest
//   earlier writers) -> ud_base_kernel (one CTA: transaction-order positions) -> ud_resolve_kernel (per key) -> ud_seg_kernel (per
//   transaction holding a wanted record: one re-scan) -> ud_compact_kernel (one CTA: order, metadata offsets, totals) -> host reads the
//   totals -> ud_emit_kernel (per record).
static int upd_build(fabgpu_ctx* ctx, int slot)
{
    auto& s = ctx->sv; auto& db = ctx->dbs[slot];
    const uint32_t R = s.upd_R, T = s.upd_T, K = s.upd_K;
    if (!s.upd_incomplete && T && memchr(s.h_flags.get(), bdev::TXC_NOT_VALIDATED, T)) s.upd_incomplete = true;    // a 254 is left
    if (s.upd_incomplete || R == 0) return FABGPU_OK;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    uint32_t P = 64;
    while (P < 2 * (uint64_t)R) P <<= 1;
    Grow g{ctx};
    g(s.d_upair, (size_t)P * sizeof(bdev::UdPair)); g(s.d_ukey, (size_t)K * sizeof(bdev::UdKey)); g(s.d_useg, (size_t)R * sizeof(bdev::UdSeg));
    g(s.d_uneed, R); g(s.d_utxneed, T); g(s.d_ubase, 4 * (size_t)T); g(s.d_umark, 4 * (size_t)R); g(s.d_uokey, 4 * (size_t)R);
    g(s.d_uomoff, 4 * (size_t)R); g(s.d_uctr, 16); g(s.h_uctr, 16);
    if (g.rc) return g.rc;
    CK(ctx, cudaMemsetAsync(s.d_upair.get(), 0, (size_t)P * sizeof(bdev::UdPair), st));
    CK(ctx, cudaMemsetAsync(s.d_ukey.get(), 0, (size_t)K * sizeof(bdev::UdKey), st));
    CK(ctx, cudaMemsetAsync(s.d_uneed.get(), 0, R, st));
    CK(ctx, cudaMemsetAsync(s.d_utxneed.get(), 0, T, st));
    CK(ctx, cudaMemsetAsync(s.d_umark.get(), 0, 4 * (size_t)R, st));
    CK(ctx, cudaMemsetAsync(s.d_uctr.get(), 0, 16, st));
    bdev::UdArrays a;
    a.rec = s.d_rec.get(); a.first_rec = s.d_first.get(); a.n_rec = s.d_n.get(); a.flags = s.d_flags.get(); a.R = R; a.T = T; a.K = K;
    a.pair = s.d_upair.get(); a.P_size = P; a.key = s.d_ukey.get(); a.base = s.d_ubase.get(); a.mark = s.d_umark.get();
    a.need = s.d_uneed.get(); a.txneed = s.d_utxneed.get(); a.seg = s.d_useg.get(); a.out_key = s.d_uokey.get(); a.out_moff = s.d_uomoff.get();
    a.out = nullptr; a.meta = nullptr; a.ctr = s.d_uctr.get();
    const uint8_t* blk = ctx->bbs[slot].d_block.get();
    bdev::ud_pair_kernel<<<(R + 255) / 256, 256, 0, st>>>(a);
    bdev::ud_class_kernel<<<P / 256 + 1, 256, 0, st>>>(a);
    bdev::ud_walk_kernel<<<P / 256 + 1, 256, 0, st>>>(a);
    bdev::ud_base_kernel<<<1, 1024, 0, st>>>(a);
    bdev::ud_resolve_kernel<<<(K + 255) / 256, 256, 0, st>>>(a);
    bdev::ud_seg_kernel<<<(T + 63) / 64, 64, 0, st>>>(blk, db.d_txs.get(), a);
    bdev::ud_compact_kernel<<<1, 1024, 0, st>>>(a);
    ctx->launches += 7;
    CK(ctx, cudaGetLastError());
    uint32_t* hc = s.h_uctr.get();
    CK(ctx, cudaMemcpyAsync(hc, s.d_uctr.get(), 12, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    if (hc[0]) { s.upd_incomplete = true; return FABGPU_OK; }
    const uint32_t n = hc[1], mb = hc[2];
    if (n) {
        Grow g2{ctx};
        g2(s.d_uout, (size_t)n * bdev::UD_WORDS * 4); g2(s.d_umeta, std::max<size_t>(mb, 1));
        if (g2.rc) return g2.rc;
        a.out = s.d_uout.get(); a.meta = s.d_umeta.get();
        bdev::ud_emit_kernel<<<(n + 127) / 128, 128, 0, st>>>(blk, a);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaStreamSynchronize(st));
    }
    s.upd_n[0] = n; s.upd_n[1] = mb;
    return FABGPU_OK;
}

int fabgpu_block_updates(fabgpu_ctx* ctx, int slot, uint64_t block_num, uint32_t* rec, size_t rec_cap, uint8_t* meta, size_t meta_cap,
                         size_t n_out[2], int* complete)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (!n_out || !complete || (rec_cap && !rec) || (meta_cap && !meta)) { ctx->last_error = "output arrays missing"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    if (s.upd_slot != slot || s.upd_block != block_num || !ctx->dbs[slot].upd_ready) {
        ctx->last_error = "no update batch for this slot and block: fabgpu_validate_mvcc(slot, block_num) last ran on another, or a stage, a "
                          "state version call or the slot's next submit came after it";
        return FABGPU_E_ARG;
    }
    if (!s.upd_built) {
        if (int rc = upd_build(ctx, slot)) return rc;
        s.upd_built = true;
    }
    n_out[0] = n_out[1] = 0; *complete = 0;
    if (s.upd_incomplete) return FABGPU_OK;
    *complete = 1; n_out[0] = s.upd_n[0]; n_out[1] = s.upd_n[1];
    const size_t w = std::min(s.upd_n[0], rec_cap), m = std::min(s.upd_n[1], meta_cap);
    if (w || m) {
        CK(ctx, cudaSetDevice(ctx->devs[0].id));
        cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
        if (w) CK(ctx, cudaMemcpyAsync(rec, s.d_uout.get(), w * bdev::UD_WORDS * 4, cudaMemcpyDeviceToHost, st));
        if (m) CK(ctx, cudaMemcpyAsync(meta, s.d_umeta.get(), m, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
    }
    return FABGPU_OK;
}

static bdev::UbArrays ubytes_arrays(fabgpu_ctx* ctx, int slot)
{
    auto& s = ctx->sv;
    bdev::UbArrays a;
    a.rec = s.d_uout.get(); a.n = (uint32_t)s.upd_n[0]; a.blk = ctx->bbs[slot].d_block.get();
    a.item = s.upd_sorted ? s.d_bitem2.get() : s.d_bitem.get(); a.cidx = s.d_bcidx.get(); a.cval = nullptr; a.coff = nullptr;
    a.block_num = s.upd_block; a.off = nullptr; a.chunk = nullptr; a.out = nullptr; a.ctr = s.d_bctr.get();
    return a;
}

// The order of a complete batch's records for fabgpu_block_update_bytes, built once per batch (on `slot`'s stream; returns
// synchronised): ub_item_kernel (per record: its sort item, whether its value is COMMITTED) -> ub_sort_kernel (one launch per merge
// pass) -> ub_cscan_kernel (one CTA: each record's index among the COMMITTED-value records) -> host reads their count.
static int ubytes_order(fabgpu_ctx* ctx, int slot)
{
    auto& s = ctx->sv;
    const uint32_t n = (uint32_t)s.upd_n[0];
    s.upd_sorted = 0; s.upd_ncom = 0;
    if (s.upd_incomplete || n == 0) return FABGPU_OK;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    Grow g{ctx};
    g(s.d_bitem, (size_t)n * sizeof(bdev::UbItem)); g(s.d_bitem2, (size_t)n * sizeof(bdev::UbItem)); g(s.d_bcidx, 4 * (size_t)n);
    g(s.d_bctr, 16); g(s.h_bctr, 16);
    if (g.rc) return g.rc;
    CK(ctx, cudaMemsetAsync(s.d_bctr.get(), 0, 16, st));
    bdev::UbArrays a = ubytes_arrays(ctx, slot);
    bdev::ub_item_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
    ctx->launches++;
    bdev::UbItem* in = s.d_bitem.get(); bdev::UbItem* out = s.d_bitem2.get();
    for (uint32_t width = 1; width < n; width <<= 1) {
        bdev::ub_sort_kernel<<<(n + 255) / 256, 256, 0, st>>>(in, out, n, width, a.blk);
        ctx->launches++;
        std::swap(in, out);
    }
    s.upd_sorted = in == s.d_bitem2.get();
    bdev::ub_cscan_kernel<<<1, 1024, 0, st>>>(a);
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(s.h_bctr.get(), s.d_bctr.get(), 8, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    s.upd_ncom = s.h_bctr.get()[1];
    return FABGPU_OK;
}

// The batch's deterministic bytes (on `slot`'s stream; returns synchronised), after ubytes_order:
//   H2D committed values -> ub_size_kernel (per sorted position: framed length, long-value chunks, UTF-8 of the names) -> ub_scan_kernel
//   (one CTA: offsets, chunk indices, totals) -> host reads the totals -> ub_emit_kernel (one warp per position) -> ub_long_kernel (one
//   CTA per chunk of the values over UB_SHORT bytes) -> D2H at most out_cap bytes.
int fabgpu_block_update_bytes(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* val_blob, const uint32_t* val_off, size_t n_val,
                              uint8_t* out, size_t out_cap, size_t* n_out, int* complete)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (!n_out || !complete || (out_cap && !out)) { ctx->last_error = "output arrays missing"; return FABGPU_E_ARG; }
    if (n_val && !val_off) { ctx->last_error = "arrays missing"; return FABGPU_E_ARG; }
    if (n_val >= UINT32_MAX) { ctx->last_error = "too many committed values for one call"; return FABGPU_E_ARG; }
    for (size_t j = 0; j < n_val; j++) if (val_off[j + 1] < val_off[j]) { ctx->last_error = "committed-value offsets decrease"; return FABGPU_E_ARG; }
    const size_t vbytes = n_val ? val_off[n_val] : 0;
    if (vbytes && !val_blob) { ctx->last_error = "arrays missing"; return FABGPU_E_ARG; }
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv;
    if (s.upd_slot != slot || s.upd_block != block_num || !ctx->dbs[slot].upd_ready) {
        ctx->last_error = "no update batch for this slot and block: fabgpu_validate_mvcc(slot, block_num) last ran on another, or a stage, a "
                          "state version call or the slot's next submit came after it";
        return FABGPU_E_ARG;
    }
    if (!s.upd_built) {
        if (int rc = upd_build(ctx, slot)) return rc;
        s.upd_built = true;
    }
    if (!s.upd_ordered) {
        if (int rc = ubytes_order(ctx, slot)) return rc;
        s.upd_ordered = true;
    }
    if (!s.upd_incomplete && n_val != s.upd_ncom) {
        ctx->last_error = "n_val is not the number of the batch's records whose value source is FABGPU_SRC_COMMITTED";
        return FABGPU_E_ARG;
    }
    *n_out = 0; *complete = 0;
    if (s.upd_incomplete) return FABGPU_OK;
    const uint32_t n = (uint32_t)s.upd_n[0];
    if (n == 0) { *complete = 1; return FABGPU_OK; }
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    Grow g{ctx};
    g(s.d_boff, 8 * ((size_t)n + 1)); g(s.d_bchunk, 4 * ((size_t)n + 1)); g(s.d_bval, std::max<size_t>(vbytes, 1));
    g(s.d_bvoff, 4 * (n_val + 1)); g(s.h_btot, 16);
    if (g.rc) return g.rc;
    if (vbytes) CK(ctx, cudaMemcpyAsync(s.d_bval.get(), val_blob, vbytes, cudaMemcpyHostToDevice, st));
    if (n_val) CK(ctx, cudaMemcpyAsync(s.d_bvoff.get(), val_off, 4 * (n_val + 1), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemsetAsync(s.d_bctr.get(), 0, 4, st));
    bdev::UbArrays a = ubytes_arrays(ctx, slot);
    a.cval = s.d_bval.get(); a.coff = s.d_bvoff.get(); a.off = s.d_boff.get(); a.chunk = s.d_bchunk.get();
    bdev::ub_size_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
    bdev::ub_scan_kernel<<<1, 1024, 0, st>>>(a);
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    unsigned long long* ht = s.h_btot.get();
    CK(ctx, cudaMemcpyAsync(ht, a.off + n, 8, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaMemcpyAsync(s.h_bctr.get(), a.chunk + n, 4, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaMemcpyAsync(s.h_bctr.get() + 1, a.ctr, 4, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    const size_t total = (size_t)ht[0]; const uint32_t chunks = s.h_bctr.get()[0];
    if (s.h_bctr.get()[1]) return FABGPU_OK;                       // a name is not UTF-8: proto.Marshal fails
    if (total) {
        Grow g2{ctx};
        g2(s.d_bout, total);
        if (g2.rc) return g2.rc;
        a.out = s.d_bout.get();
        bdev::ub_emit_kernel<<<(uint32_t)(((size_t)n * 32 + 255) / 256), 256, 0, st>>>(a);
        ctx->launches++;
        if (chunks) { bdev::ub_long_kernel<<<chunks, 256, 0, st>>>(a); ctx->launches++; }
        CK(ctx, cudaGetLastError());
        const size_t w = std::min(total, out_cap);
        if (w) CK(ctx, cudaMemcpyAsync(out, s.d_bout.get(), w, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
    }
    *n_out = total; *complete = 1;
    return FABGPU_OK;
}

// Builds the private update batch after pvt_check left its records on the device (on `slot`'s stream; returns synchronised).  complete:
// 0 when the peer builds it itself; n_rec: the records, whose words are in p.h_out.
//   pu_list_kernel (per entry: writes and metadata writes of a VALID entry that passed; the host reads the counts, grows the arrays and
//   runs it again on overflow) -> sha256_segments_kernel (per metadata write: its key) -> pu_base_kernel (one CTA: transaction-order
//   positions) -> pu_key_kernel (per item: the key table, the last writer) -> pu_first_kernel (per item) -> pu_renew_kernel (per
//   metadata write: the hashed record, the value to compare) -> sha256_segments_kernel (per metadata write: that value) -> pu_mark_kernel
//   (per key) -> pu_compact_kernel (one CTA: order, totals) -> host reads the totals -> pu_emit_kernel (per record).
static int pvu_build(fabgpu_ctx* ctx, int slot, uint32_t E, uint32_t T, int& complete, size_t& n_rec)
{
    auto& s = ctx->sv; auto& p = ctx->pvt[slot];
    complete = 0; n_rec = 0;
    cudaStream_t st = ctx->devs[0].slot[slot].stream.get();
    const uint32_t K = s.upd_n[0] ? s.upd_K : 0, H = (uint32_t)s.upd_n[0];
    Grow grow{ctx};
    grow(p.d_wfirst, 4 * (size_t)E); grow(p.d_mfirst, 4 * (size_t)E); grow(p.d_tbase, 4 * (size_t)T); grow(p.d_pctr, 32); grow(p.h_pctr, 32);
    grow(p.d_rmark, 4 * (size_t)std::max(K, 1u));
    if (grow.rc) return grow.rc;
    bdev::PuArrays a;
    a.pvt = p.d_blob.get(); a.seq = p.d_seq.get(); a.n_pvt = E; a.T = T; a.flags = p.d_flags.get(); a.status = p.d_status.get();
    a.rec = p.d_rec.get(); a.first = p.d_first.get(); a.n_rec = p.d_n.get(); a.wfirst = p.d_wfirst.get(); a.mfirst = p.d_mfirst.get();
    a.tbase = p.d_tbase.get(); a.ctr = p.d_pctr.get(); a.seed = s.seed; a.stage_seed = s.seed; a.blk = ctx->bbs[slot].d_block.get();
    a.stage.key = K ? s.d_key.get() : nullptr; a.stage.K_size = K;
    a.ukey = K ? s.d_ukey.get() : nullptr; a.useg = K ? s.d_useg.get() : nullptr; a.uokey = K ? s.d_uokey.get() : nullptr; a.n_h = H;
    a.rmark = p.d_rmark.get();
    uint32_t* hc = p.h_pctr.get();
    uint32_t W = 0, M = 0;
    for (;;) {
        const size_t W_cap = (size_t)E * p.w_hint, M_cap = (size_t)E * p.m_hint;
        if (W_cap > UINT32_MAX || M_cap > UINT32_MAX) { ctx->last_error = "too many private writes for one call"; return FABGPU_E_ARG; }
        Grow g2{ctx};
        g2(p.d_item, W_cap * sizeof(bdev::PuItem)); g2(p.d_meta, M_cap * sizeof(bdev::PuItem)); g2(p.d_mjobs, M_cap * sizeof(bdev::ShaJobP));
        g2(p.d_mdig, 32 * M_cap);
        if (g2.rc) return g2.rc;
        a.item = p.d_item.get(); a.W_cap = (uint32_t)W_cap; a.meta = p.d_meta.get(); a.M_cap = (uint32_t)M_cap; a.jobs = p.d_mjobs.get();
        a.dig = p.d_mdig.get();
        CK(ctx, cudaMemsetAsync(p.d_tbase.get(), 0, 4 * (size_t)T, st));
        CK(ctx, cudaMemsetAsync(p.d_pctr.get(), 0, 32, st));
        bdev::pu_list_kernel<<<(E + 63) / 64, 64, 0, st>>>(a);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(hc, p.d_pctr.get(), 12, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
        W = hc[0]; M = hc[1];
        if (W <= W_cap && M <= M_cap) break;
        if (W > W_cap) p.w_hint = (uint32_t)((W + E - 1) / E) + 1;        // later calls are sized for it too
        if (M > M_cap) p.m_hint = (uint32_t)((M + E - 1) / E) + 1;
    }
    if (hc[2]) return FABGPU_OK;                                         // a Put of a nil value
    uint32_t P = 64;
    while (P < 2 * ((uint64_t)W + M)) P <<= 1;
    Grow g3{ctx};
    g3(p.d_key, (size_t)P * sizeof(bdev::PuKey)); g3(p.d_mark, 4 * (size_t)std::max(W, 1u)); g3(p.d_okey, 4 * ((size_t)W + H + 1));
    if (g3.rc) return g3.rc;
    a.key = p.d_key.get(); a.P_size = P; a.mark = p.d_mark.get(); a.out_key = p.d_okey.get();
    CK(ctx, cudaMemsetAsync(p.d_key.get(), 0, (size_t)P * sizeof(bdev::PuKey), st));
    CK(ctx, cudaMemsetAsync(p.d_mark.get(), 0, 4 * (size_t)std::max(W, 1u), st));
    if (K) CK(ctx, cudaMemsetAsync(p.d_rmark.get(), 0, 4 * (size_t)K, st));
    const ShaJob* jobs = reinterpret_cast<const ShaJob*>(p.d_mjobs.get());
    if (M) { sha256_segments_kernel<<<(M + 127) / 128, 128, 0, st>>>(p.d_blob.get(), jobs, M, p.d_mdig.get()); ctx->launches++; }
    bdev::pu_base_kernel<<<1, 1024, 0, st>>>(a);
    ctx->launches++;
    if (W + M) {
        bdev::pu_key_kernel<<<(W + M + 255) / 256, 256, 0, st>>>(a, W, W + M);
        bdev::pu_first_kernel<<<(W + M + 255) / 256, 256, 0, st>>>(a, W, W + M);
        ctx->launches += 2;
    }
    if (M) {
        bdev::pu_renew_kernel<<<(M + 127) / 128, 128, 0, st>>>(a, M);
        sha256_segments_kernel<<<(M + 127) / 128, 128, 0, st>>>(p.d_blob.get(), jobs, M, p.d_mdig.get());
        ctx->launches += 2;
    }
    bdev::pu_mark_kernel<<<P / 256 + 1, 256, 0, st>>>(a);
    bdev::pu_compact_kernel<<<1, 1024, 0, st>>>(a, W);
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(hc, p.d_pctr.get(), 20, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    if (hc[2]) return FABGPU_OK;
    const size_t n = (size_t)hc[3] + hc[4];
    if (n) {
        Grow g4{ctx};
        g4(p.d_out, n * bdev::PU_WORDS * 4); g4(p.h_out, n * bdev::PU_WORDS * 4);
        if (g4.rc) return g4.rc;
        a.out = p.d_out.get();
        bdev::pu_emit_kernel<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>(a);
        ctx->launches++;
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(p.h_out.get(), p.d_out.get(), n * bdev::PU_WORDS * 4, cudaMemcpyDeviceToHost, st));
        CK(ctx, cudaStreamSynchronize(st));
    }
    complete = 1; n_rec = n;
    return FABGPU_OK;
}

int fabgpu_block_pvt_updates(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* pvt_blob, const uint32_t* pvt_off, const uint32_t* seq,
                             size_t n_pvt, int32_t* status, int32_t out[4], uint32_t* rec, size_t rec_cap, size_t* n_out, int* complete)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (!out || !n_out || !complete || (rec_cap && !rec)) { ctx->last_error = "output arrays missing"; return FABGPU_E_ARG; }
    if (n_pvt && (!pvt_off || !seq || !status)) { ctx->last_error = "arrays missing"; return FABGPU_E_ARG; }
    if (int rc = pvt_args(ctx, pvt_blob, pvt_off, n_pvt)) return rc;
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    auto& s = ctx->sv; auto& db = ctx->dbs[slot];
    if (s.upd_slot != slot || s.upd_block != block_num || !db.upd_ready) {
        ctx->last_error = "no update batch for this slot and block: fabgpu_validate_mvcc(slot, block_num) last ran on another, or a stage, a "
                          "state version call or the slot's next submit came after it";
        return FABGPU_E_ARG;
    }
    const size_t n = db.T;
    if (int rc = pvt_seqs(ctx, seq, n_pvt, n)) return rc;
    if (!s.upd_built) {
        if (int rc = upd_build(ctx, slot)) return rc;
        s.upd_built = true;
    }
    *n_out = 0; *complete = 0;
    uint32_t R;
    if (int rc = pvt_check(ctx, slot, s.upd_flags.data(), n, pvt_blob, pvt_off, seq, n_pvt, status, out, R)) return rc;
    if (s.upd_incomplete || out[0] != bdev::PV_OK) return FABGPU_OK;
    if (n_pvt == 0) { *complete = 1; return FABGPU_OK; }
    int c = 0; size_t nr = 0;
    if (int rc = pvu_build(ctx, slot, (uint32_t)n_pvt, (uint32_t)n, c, nr)) return rc;
    if (!c) return FABGPU_OK;
    *complete = 1; *n_out = nr;
    const size_t w = std::min(nr, rec_cap);
    if (w) memcpy(rec, ctx->pvt[slot].h_out.get(), w * bdev::PU_WORDS * 4);
    return FABGPU_OK;
}

int fabgpu_block_buffer_slot(fabgpu_ctx* ctx, int slot, size_t bytes, uint8_t** out)
{
    if (!ctx || !out || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    auto& bb = ctx->bbs[slot];
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    if (bytes > bb.h_block.bytes() && ctx->dbs[slot].busy) { ctx->last_error = "slot holds a block in flight"; return FABGPU_E_ARG; }
    if (int rc = bb.h_block.reserve(ctx, bytes)) return rc;
    *out = bb.h_block.get();
    return FABGPU_OK;
}
int fabgpu_block_buffer(fabgpu_ctx* ctx, size_t bytes, uint8_t** out) { return fabgpu_block_buffer_slot(ctx, 0, bytes, out); }

// Device path of the block pre-pass: the host only copies bytes in and flags out (and marks duplicate tx ids).
//   H2D block + envelope offsets -> block_walk_kernel (per transaction) -> block_resolve_kernel (per signature: identity lookup, DER gates)
//   -> sha256_segments_kernel (signed messages + check digests) -> one verify launch -> block_decide_kernel -> D2H flags.
// Everything is enqueued on the slot's stream in one go: the number of endorsement jobs (known only after the walk) stays
// on the device -- the later launches are sized for the worst case and read the count themselves.
static int block_submit(fabgpu_ctx* ctx, int slot, const uint8_t* block, size_t block_len, const uint32_t* env_off, size_t n_env)
{
    auto now = [] { return std::chrono::steady_clock::now(); };
    Device& dv = ctx->devs[0];
    DevSlot& ds = dv.slot[slot];
    auto& bb = ctx->bbs[slot]; auto& db = ctx->dbs[slot]; auto& dm = ctx->dm;
    db.t0 = now();
    CK(ctx, cudaSetDevice(dv.id));
    // Identities' key tables may have been recycled by other registrations since fabgpu_msp_configure, in this context or another of
    // its group: re-issue them.  From the check to the last enqueue of this block the slot table is held shared (KeyTables::tab_mu): a
    // concurrent fabgpu_keys_register in any context of the group waits, so dm.key_slot's raw slots stay the tables of these identities for the whole launch sequence.
    std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);
    {
        auto any_stale = [&] {
            std::lock_guard<std::mutex> lk(ctx->mu);
            for (size_t i = 0; i < ctx->identity_slot.size(); i++)
                if (ctx->identity_slot[i] != -1 && handle_to_slot(ctx, ctx->identity_slot[i]) == -1) return true;
            return false;
        };
        if (any_stale()) {
            rl.unlock();
            // every identity in its own tier (fabgpu_ctx::identity_tier): configured ones as fabgpu_msp_configure issued them, admitted ones small
            const int n_ids = (int)ctx->identity_slot.size();
            for (uint8_t tier : {TIER_WINDOW, TIER_SMALL}) {
                std::vector<int> which;
                for (int i = 0; i < n_ids; i++) if (ctx->identity_tier[i] == tier) which.push_back(i);
                if (which.empty()) continue;
                const int m = (int)which.size();
                std::vector<uint8_t> keys(64 * (size_t)m);
                std::vector<int32_t> hd(m);
                for (int q = 0; q < m; q++) { memcpy(keys.data() + 64 * (size_t)q, ctx->msp.keys_xy.data() + 64 * (size_t)which[q], 64); hd[q] = ctx->identity_slot[which[q]]; }
                int rc = tier == TIER_WINDOW ? fabgpu_keys_register(ctx, keys.data(), m, hd.data())     // exclusive; drains every stream first
                                             : msp_small_tier(ctx, keys.data(), m, hd.data());
                if (rc) return rc;
                for (int q = 0; q < m; q++) ctx->identity_slot[which[q]] = hd[q];
            }
            rl.lock();
            std::vector<int32_t> raw(n_ids > 0 ? n_ids : 1, -1);
            dm.all_slots = true; dm.classes = 0;
            msp_raw_slots(ctx, 0, n_ids, raw.data());         // a handle recycled again in the gap resolves to -1: that identity goes through the generic kernel
            // submitters are serialised by slot0_mu; blocks in flight on the other slots still read dm.key_slot, and admissions write it:
            // let them finish first
            for (auto& dsx : dv.slot) CK(ctx, cudaStreamSynchronize(dsx.stream.get()));
            if (ctx->adm.stream) CK(ctx, cudaStreamSynchronize(ctx->adm.stream.get()));
            CK(ctx, cudaMemcpy(dm.key_slot.get(), raw.data(), 4 * (size_t)n_ids, cudaMemcpyHostToDevice));
        }
    }
    // The slot's last fabgpu_committed_txids_add_block may still be reading its block and envelope table (TxidSet::read_ev): a buffer
    // is reallocated only after that kernel has finished, and the copies below are enqueued behind it.
    auto& tx_set = ctx->txid;
    auto txid_read_done = [&]() -> int {
        if (tx_set.read_set[slot]) CK(ctx, cudaEventSynchronize(tx_set.read_ev[slot].get()));
        tx_set.read_set[slot] = false;
        return FABGPU_OK;
    };
    // slack: word-wise readers (bytes_equal, the SHA loader) touch the aligned words past the end.  An empty block needs no buffer.
    if (block_len && block_len + 64 > bb.d_block.bytes()) {
        if (int rc = txid_read_done()) return rc;
        if (int rc = bb.d_block.reserve(ctx, block_len + (block_len >> 2) + 64)) return rc;
    }
    const char* evs = getenv("FABGPU_BLOCK_EVENTS");          // "1": time the device stages with CUDA events (diagnostics)
    db.use_ev = evs && evs[0] == '1';
    if (db.use_ev) for (auto& e : db.ev) if (!e) { cudaEvent_t ev = nullptr; CK(ctx, cudaEventCreate(&ev)); e.reset(ev); }
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[0].get(), ds.stream.get()));
    std::vector<uint32_t> split;
    if (!env_off) {                                           // serialized common.Block: find the envelopes (serial, length-prefixed)
        std::vector<blockval::Seg> envs;
        if (!blockval::split_block(block, block_len, envs)) { ctx->last_error = "block does not parse"; return FABGPU_E_ARG; }
        n_env = envs.size();
        split.resize(2 * n_env + 2);
        for (size_t i = 0; i < n_env; i++) { split[2 * i] = envs[i].off; split[2 * i + 1] = envs[i].off + envs[i].len; }
    }
    if (dm.nodes_lost) { ctx->last_error = "policy nodes lost by a failed fabgpu_key_policies call: call fabgpu_msp_configure again"; return FABGPU_E_CUDA; }
    const size_t T = n_env;
    db.T = T; db.block = block;
    if (T == 0) return FABGPU_OK;
    const size_t J_cap = T * (1 + BD_ENDS_HINT);
    if (T > db.tx_cap()) {
        if (int rc = txid_read_done()) return rc;
        const size_t tc = T + (T >> 2) + 256, jc = tc * (1 + BD_ENDS_HINT);
        Grow grow{ctx};
        grow(db.d_env_off, 8 * (tc + 1)); grow(db.d_txs, sizeof(bdev::TxDev) * tc);
        grow(db.d_raw, sizeof(bdev::RawJob) * jc);
        grow(db.d_sha, sizeof(bdev::ShaJobD) * (jc + 2 * tc)); grow(db.d_dig, 32 * (jc + 2 * tc) + 64);
        grow(db.d_r, 32 * jc); grow(db.d_s, 32 * jc); grow(db.d_qx, 32 * jc); grow(db.d_qy, 32 * jc);
        grow(db.d_gate, jc); grow(db.d_ks, 4 * jc); grow(db.d_ident, 4 * jc);
        grow(db.d_mask, jc / 8 + 8); grow(db.d_off, jc / 8 + 8); grow(db.d_counter, 16); grow(db.d_idx, 4 * (jc + 2));
        grow(db.d_scal, 64 * jc);
        grow(db.d_flags, tc); grow(db.d_hash, 8 * tc); grow(db.d_seg, 8 * tc);
        grow(db.h_hash, 8 * tc); grow(db.h_seg, 8 * tc); grow(db.h_counter, 16); grow(db.h_env_off, 8 * (tc + 1));
        grow(db.h_flags, tc);
        if (grow.rc) return grow.rc;
    }
    // envelope table on the device: pairs (begin, end) so that both entry points share one kernel
    for (size_t i = 0; i < T; i++) {
        db.h_env_off.get()[2 * i] = env_off ? env_off[i] : split[2 * i];
        db.h_env_off.get()[2 * i + 1] = env_off ? env_off[i + 1] : split[2 * i + 1];
    }
    cudaStream_t st = ds.stream.get();
    if (tx_set.read_set[slot]) {
        CK(ctx, cudaStreamWaitEvent(st, tx_set.read_ev[slot].get(), 0));
        tx_set.read_set[slot] = false;
    }
    CK(ctx, cudaMemcpyAsync(db.d_env_off.get(), db.h_env_off.get(), 8 * T, cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemsetAsync(db.d_counter.get(), 0, 16, st));
    bdev::MspDev m; m.id_blob = dm.id_blob.get(); m.id_off = dm.id_off.get(); m.key_slot = dm.key_slot.get(); m.valid = dm.valid.get(); m.msp_code = dm.msp_code.get(); m.group = dm.group.get();
    m.keys_xy = dm.keys_xy.get(); m.ht_hash = dm.ht_hash.get(); m.ht_idx = dm.ht_idx.get(); m.ht_size = dm.ht_size; m.n_ids = dm.n_ids;
    bdev::PolicyDev pol; pol.nodes = dm.nodes.get(); pol.n_nodes = dm.n_nodes; pol.principal_code = dm.principal_code.get(); pol.n_principals = dm.n_principals;
    pol.ns_blob = dm.ns_blob.get(); pol.ns_off = dm.ns_off.get(); pol.ns_root = dm.ns_root.get(); pol.n_ns = dm.n_ns;
    pol.principal_bits = dm.pbits.get(); pol.bits_words = dm.pbits_words;
    pol.coll_ns_blob = dm.cp_ns_blob.get(); pol.coll_ns_off = dm.cp_ns_off.get(); pol.coll_name_blob = dm.cp_name_blob.get(); pol.coll_name_off = dm.cp_name_off.get();
    pol.coll_root = dm.cp_root.get(); pol.coll_hash = dm.cp_hash.get(); pol.coll_idx = dm.cp_idx.get(); pol.coll_size = dm.cp_size;
    pol.n_nodes = dm.n_nodes + dm.kp_n_nodes; pol.kp_slots = dm.kp_slots.get(); pol.kp_blob = dm.kp_blob.get(); pol.kp_size = dm.kp_size;
    pol.mode = dm.mode; pol.ver_blob = dm.ver_blob.get(); pol.ver_off = dm.ver_off.get();
    db.v13 = dm.mode == BD_MODE_V13;
    bdev::KlArrays kl;                                        // key policy table installed: write records and the metadata-write set
    db.kl_on = dm.kp_size != 0;
    if (db.kl_on) {
        const size_t W_cap = T * ctx->kl_hint.load();
        size_t md = 64; while (md < 2 * W_cap) md <<= 1;
        Grow grow{ctx};
        grow(db.d_w, sizeof(bdev::WriteRec) * W_cap); grow(db.d_md_hash, 8 * md); grow(db.d_clist, 4 * T); grow(db.d_conf, T);
        grow(db.d_md_min, 8 * md); grow(db.d_md_sum, 4 * md);
        if (grow.rc) return grow.rc;
        CK(ctx, cudaMemsetAsync(db.d_md_hash.get(), 0, 8 * md, ds.stream.get()));
        CK(ctx, cudaMemsetAsync(db.d_md_min.get(), 0xff, 8 * md, ds.stream.get()));
        CK(ctx, cudaMemsetAsync(db.d_md_sum.get(), 0, 4 * md, ds.stream.get()));
        kl.w = db.d_w.get(); kl.W_cap = (uint32_t)W_cap; kl.counter = db.d_counter.get() + 2; kl.md_hash = db.d_md_hash.get();
        kl.md_min = db.d_md_min.get(); kl.md_sum = db.d_md_sum.get(); kl.md_size = (uint32_t)md; kl.conflicted = db.d_conf.get(); kl.clist = db.d_clist.get();
        db.W_cap = W_cap;
    }
    const bool need_q = (dm.classes & CLASS_GENERIC) != 0;   // only the generic arithmetic reads the key itself
    bdev::JobArrays ja; ja.sha = db.d_sha.get(); ja.r = db.d_r.get(); ja.s = db.d_s.get(); ja.key_slot = db.d_ks.get(); ja.identity = db.d_ident.get(); ja.qx = need_q ? db.d_qx.get() : nullptr;
    ja.qy = need_q ? db.d_qy.get() : nullptr; ja.gate_ok = db.d_gate.get(); ja.J_cap = (uint32_t)J_cap; ja.T = (uint32_t)T; ja.kl = kl; ja.mode = dm.mode;
    const uint32_t cnt = (uint32_t)T, E_cap = (uint32_t)(J_cap - T);
    // One copy, then the walk.  (Copying in chunks with a walk per chunk was measured slower, the more chunks the slower: hashing a
    // 4.6 KB payload is a long chain of dependent rounds per thread however few
    // threads a launch has, so per-chunk launches serialise that latency.  What hides the copy is the NEXT block's copy running
    // under this block's kernels: the slots.)
    CK(ctx, cudaMemcpyAsync(bb.d_block.get(), block, block_len, cudaMemcpyHostToDevice, st));
    bdev::block_walk_kernel<<<(cnt + 31) / 32, 32, 0, st>>>(bb.d_block.get(), db.d_env_off.get(), 0u, cnt, cnt, dm.channel.get(), dm.channel_len, db.d_txs.get(), db.d_raw.get(), ja, db.d_counter.get());
    if (ctx->adm.ev_set) CK(ctx, cudaStreamWaitEvent(st, ctx->adm.ev.get(), 0));      // the MSP table as the admissions returned so far left it
    bdev::block_resolve_kernel<<<(cnt + 63) / 64, 64, 0, st>>>(bb.d_block.get(), db.d_raw.get(), 0u, cnt, m, ja, db.d_txs.get());                      // creator jobs
    sha256_segments_kernel<<<(cnt + 127) / 128, 128, 0, st>>>(bb.d_block.get(), reinterpret_cast<const ShaJob*>(db.d_sha.get()), cnt, db.d_dig.get());
    sha256_segments_kernel<<<(2 * cnt + 127) / 128, 128, 0, st>>>(bb.d_block.get(), reinterpret_cast<const ShaJob*>(db.d_sha.get() + J_cap), 2 * cnt, db.d_dig.get() + 32 * J_cap);
    ctx->launches += 4;
    CK(ctx, cudaGetLastError());
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[1].get(), st));
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[2].get(), st));
    // endorsement jobs [T, T + *d_counter): launches sized for the worst case, the kernels stop at the device-side count
    bdev::block_resolve_kernel<<<(E_cap + 63) / 64, 64, 0, st>>>(bb.d_block.get(), db.d_raw.get(), cnt, E_cap, m, ja, db.d_txs.get(), db.d_counter.get());
    sha256_segments_kernel<<<(E_cap + 127) / 128, 128, 0, st>>>(bb.d_block.get(), reinterpret_cast<const ShaJob*>(db.d_sha.get()) + T, E_cap, db.d_dig.get() + 32 * T, db.d_counter.get());
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[3].get(), st));
    int rc = launch_verify(ctx, dv, dm.all_slots ? MODE_CACHED : MODE_MIXED, db.d_ks.get(), db.d_qx.get(), db.d_qy.get(), db.d_dig.get(), db.d_r.get(), db.d_s.get(), J_cap, db.d_mask.get(), db.d_off.get(), st,
                           db.d_counter.get(), cnt, nullptr, db.d_idx.get(), dm.classes ? dm.classes : CLASS_GENERIC, db.d_scal.get());
    if (rc) return rc;
    // the committed tx-id set as the mutations returned so far left it (all of them, as submitters and mutations hold slot0_mu)
    bdev::TxidSetDev tsd{nullptr, 0, 0, 0};
    if (tx_set.installed) {
        tsd.slots = tx_set.table; tsd.mask = (uint32_t)(tx_set.slots - 1); tsd.seed = tx_set.seed; tsd.broken = tx_set.broken || !tx_set.table;
        if (tx_set.ev_set) CK(ctx, cudaStreamWaitEvent(st, tx_set.ev.get(), 0));
    }
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[4].get(), st));
    bdev::block_decide_kernel<<<(cnt + 127) / 128, 128, 0, st>>>(bb.d_block.get(), db.d_txs.get(), cnt, m, pol, db.d_mask.get(), db.d_gate.get(), db.d_ident.get(), db.d_dig.get(), (uint32_t)J_cap, db.d_flags.get(),
                                                               db.d_hash.get(), db.d_seg.get(), kl, db.v13 ? db.d_counter.get() + 1 : nullptr, tsd);
    ctx->launches++;
    if (tx_set.installed || ctx->adm.admitted) {              // a later mutation of the set or the MSP table waits for this decide stage
        if (!tx_set.decide_ev[slot]) { cudaEvent_t ev = nullptr; CK(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); tx_set.decide_ev[slot].reset(ev); }
        CK(ctx, cudaEventRecord(tx_set.decide_ev[slot].get(), st));
        tx_set.decide_set[slot] = true;
    } else {
        tx_set.decide_set[slot] = false;                      // this block recorded none: a mutation waits for the slot's whole stream
    }
    if (db.kl_on) {
        bdev::block_kl_resolve_kernel<<<1, 256, 0, st>>>(db.d_txs.get(), cnt, kl, db.d_flags.get());
        ctx->launches++;
    }
    // [1]: an lscc invocation was flagged 254 (v1.3 mode); [2]: write records used (key policy table)
    if (db.kl_on || db.v13) CK(ctx, cudaMemcpyAsync(db.h_counter.get(), db.d_counter.get(), 16, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaGetLastError());
    if (db.use_ev) CK(ctx, cudaEventRecord(db.ev[5].get(), st));
    CK(ctx, cudaMemcpyAsync(db.h_flags.get(), db.d_flags.get(), T, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaMemcpyAsync(db.h_hash.get(), db.d_hash.get(), 8 * T, cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaMemcpyAsync(db.h_seg.get(), db.d_seg.get(), 8 * T, cudaMemcpyDeviceToHost, st));
    db.t1 = now();
    return FABGPU_OK;
}

// Waits for the slot's block and finishes on the host: markTXIdDuplicates (v20/validator.go:283-297) -- among VALID
// transactions, a later one with an already seen tx id.  Reads the caller's block bytes to confirm equal hashes.
static int block_finish(fabgpu_ctx* ctx, int slot, uint8_t* flags)
{
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::micro>(b - a).count();
    };
    auto& db = ctx->dbs[slot];
    const size_t T = db.T;
    const uint8_t* block = db.block;
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    CK(ctx, cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get()));
    auto t3 = now();
    if (T == 0) return FABGPU_OK;
    memcpy(flags, db.h_flags.get(), T);
    if (db.kl_on && db.h_counter.get()[2] > db.W_cap) {        // write records overflowed (that block's flags say 254): size later blocks for it
        const uint32_t want = (uint32_t)((db.h_counter.get()[2] + T - 1) / T) + 1;
        uint32_t cur = ctx->kl_hint.load();
        while (cur < want && !ctx->kl_hint.compare_exchange_weak(cur, want)) {}
    }
    {
        // flat open-addressing table keyed by the 64-bit tx-id hash (0 = empty); equal hashes are confirmed on the bytes
        size_t cap = 16; while (cap < 4 * T) cap <<= 1;
        db.dup_keys.assign(cap, 0); db.dup_idx.resize(cap);
        uint64_t* keys = db.dup_keys.data(); uint32_t* idx = db.dup_idx.data();
        for (size_t t = 0; t < T; t++) {
            if (flags[t] != blockval::TX_VALID) continue;
            const bdev::Seg id = db.h_seg.get()[t];
            const uint64_t h = db.h_hash.get()[t] ? db.h_hash.get()[t] : 1;
            bool dup = false;
            size_t pos = (size_t)h & (cap - 1);
            for (;; pos = (pos + 1) & (cap - 1)) {
                if (keys[pos] == 0) break;
                if (keys[pos] != h) continue;
                const bdev::Seg o = db.h_seg.get()[idx[pos]];
                if (o.len == id.len && memcmp(block + o.off, block + id.off, id.len) == 0) { dup = true; break; }
            }
            if (dup) flags[t] = blockval::TX_DUPLICATE_TXID;
            else { keys[pos] = h; idx[pos] = (uint32_t)t; }
        }
    }
    // v1.3 mode, a block with an lscc invocation flagged 254 (lscc_mark): the reference invalidates the still-VALID invocations of a chaincode an upgrade of the
    // block names (CHAINCODE_VERSION_CONFLICT, v14/validator.go:210-220,487-530); the device does not decide the upgrade, so every
    // VALID transaction goes to the CPU validator.  After the duplicate pass and the key-level resolve stage, and fed into neither.
    if (db.v13 && db.h_counter.get()[1])
        for (size_t t = 0; t < T; t++) if (flags[t] == blockval::TX_VALID) flags[t] = bdev::TXC_NOT_VALIDATED;
    auto t4 = now();
    ctx->block_timing[0] = us(db.t0, db.t1); ctx->block_timing[1] = 0; ctx->block_timing[2] = us(db.t1, t3); ctx->block_timing[3] = us(t3, t4);
    ctx->block_timing[4] = us(db.t0, t4);
    for (int k = 0; k < 5; k++) { float ms = 0; if (db.use_ev) cudaEventElapsedTime(&ms, db.ev[k].get(), db.ev[k + 1].get()); ctx->block_timing[5 + k] = 1e3 * ms; }
    return FABGPU_OK;
}

// serialized: 1 = `block` is a serialized common.Block (env_off unused), 0 = concatenated envelopes with an offset table
static int validate_submit(fabgpu_ctx* ctx, int slot, const uint8_t* block, size_t block_len, const uint32_t* env_off, size_t n_env)
{
    if (!ctx || !block || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
    if (block_len >= (1ull << 32)) { ctx->last_error = "block larger than 4 GiB"; return FABGPU_E_ARG; }
    if (env_off) {                                            // the table must be non-decreasing and stay inside the blob
        for (size_t i = 0; i < n_env; i++)
            if (env_off[i] > env_off[i + 1]) { ctx->last_error = "envelope offsets are not non-decreasing"; return FABGPU_E_ARG; }
        if (n_env && env_off[n_env] > block_len) { ctx->last_error = "envelope offsets exceed the blob length"; return FABGPU_E_ARG; }
    }
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    auto& db = ctx->dbs[slot];
    if (db.busy) { ctx->last_error = "slot already holds a block: call fabgpu_validate_wait first"; return FABGPU_E_ARG; }
    db.mvcc_ready = false; db.pvt_ready = false; db.txid_block = 0; db.upd_ready = false;
    if (fault_injected()) { ctx->last_error = "fault injected (FABGPU_FAULT_INJECT=1)"; return FABGPU_E_INJECTED; }
    int rc;
    {
        std::lock_guard<std::mutex> lk0(ctx->slot0_mu);      // key-cache / MSP state: one submitter at a time
        rc = block_submit(ctx, slot, block, block_len, env_off, n_env);
        if (rc) { cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get()); return rc; }
        db.on_device = true;
    }
    db.busy = true; db.txid_block = 1;
    return FABGPU_OK;
}

int fabgpu_validate_block_async(fabgpu_ctx* ctx, int slot, const uint8_t* block, size_t block_len)
{
    return validate_submit(ctx, slot, block, block_len, nullptr, 0);
}

int fabgpu_validate_envelopes_async(fabgpu_ctx* ctx, int slot, const uint8_t* blob, const uint32_t* env_off, size_t n_env)
{
    if (!env_off && n_env) return FABGPU_E_ARG;
    if (n_env == 0) {                                         // nothing to do, but keep the slot protocol
        if (!ctx || slot < 0 || slot >= FABGPU_SLOTS) return FABGPU_E_ARG;
        std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
        auto& db = ctx->dbs[slot];
        if (db.busy) { ctx->last_error = "slot already holds a block: call fabgpu_validate_wait first"; return FABGPU_E_ARG; }
        db.T = 0; db.on_device = false; db.busy = true; db.mvcc_ready = false; db.pvt_ready = false; db.txid_block = 1; db.upd_ready = false;
        return FABGPU_OK;
    }
    return validate_submit(ctx, slot, blob, env_off[n_env], env_off, n_env);
}

int fabgpu_validate_wait(fabgpu_ctx* ctx, int slot, uint8_t* flags, size_t flags_cap, size_t* n_tx_out)
{
    if (!ctx || slot < 0 || slot >= FABGPU_SLOTS || !n_tx_out) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->blk_mu[slot]);
    auto& db = ctx->dbs[slot];
    if (!db.busy) { ctx->last_error = "no block in flight on this slot"; return FABGPU_E_ARG; }
    db.busy = false;
    *n_tx_out = db.T;
    if (db.T > flags_cap || (db.T && !flags)) {
        if (db.on_device) cudaStreamSynchronize(ctx->devs[0].slot[slot].stream.get());
        ctx->last_error = "flags buffer too small";
        return FABGPU_E_ARG;
    }
    const int rc = db.on_device ? block_finish(ctx, slot, flags) : FABGPU_OK;      // (an empty envelope list: nothing ran)
    db.mvcc_ready = db.pvt_ready = rc == FABGPU_OK;
    return rc;
}

int fabgpu_validate_block(fabgpu_ctx* ctx, const uint8_t* block, size_t block_len, uint8_t* flags, size_t flags_cap, size_t* n_tx_out)
{
    if (!ctx || !block || !flags || !n_tx_out) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->sync_blk_mu);
    int rc = fabgpu_validate_block_async(ctx, 0, block, block_len);
    if (rc) return rc;
    return fabgpu_validate_wait(ctx, 0, flags, flags_cap, n_tx_out);
}

int fabgpu_validate_envelopes(fabgpu_ctx* ctx, const uint8_t* blob, const uint32_t* env_off, size_t n_env, uint8_t* flags, size_t flags_cap,
                              size_t* n_tx_out)
{
    if (!ctx || !blob || !env_off || !flags || !n_tx_out) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->sync_blk_mu);
    int rc = fabgpu_validate_envelopes_async(ctx, 0, blob, env_off, n_env);
    if (rc) return rc;
    return fabgpu_validate_wait(ctx, 0, flags, flags_cap, n_tx_out);
}

int fabgpu_block_timing(const fabgpu_ctx* ctx, double out_us[10])
{
    if (!ctx || !out_us) return FABGPU_E_ARG;
    for (int i = 0; i < 10; i++) out_us[i] = ctx->block_timing[i];
    return FABGPU_OK;
}

// digests[j] = SHA-256(buf[off0..) || buf[off1..) || buf[off2..)) on the device; jobs: n x 6 uint32 (off0,off1,off2,len0,len1,len2)
int fabgpu_sha256_segments(fabgpu_ctx* ctx, const uint8_t* buf, size_t buf_len, const uint32_t* jobs, size_t n, uint8_t* digests)
{
    if (!ctx || !buf || !jobs || !digests) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk0(ctx->slot0_mu);
    Device& dv = ctx->devs[0];
    CK(ctx, cudaSetDevice(dv.id));
    DevArray<uint8_t> d_buf, d_dig; DevArray<ShaJob> d_jobs;
    Grow grow{ctx};
    grow(d_buf, buf_len ? buf_len : 1); grow(d_jobs, sizeof(ShaJob) * (n ? n : 1)); grow(d_dig, 32 * (n ? n : 1));
    if (grow.rc) return grow.rc;
    CK(ctx, cudaMemcpy(d_buf.get(), buf, buf_len, cudaMemcpyHostToDevice));
    CK(ctx, cudaMemcpy(d_jobs.get(), jobs, sizeof(ShaJob) * n, cudaMemcpyHostToDevice));
    if (n) {
        sha256_segments_kernel<<<(unsigned)((n + 127) / 128), 128>>>(d_buf.get(), d_jobs.get(), (uint32_t)n, d_dig.get());
        ctx->launches++;
        CK(ctx, cudaGetLastError());
    }
    CK(ctx, cudaMemcpy(digests, d_dig.get(), 32 * n, cudaMemcpyDeviceToHost));
    return FABGPU_OK;
}

int fabgpu_test_fieldop(fabgpu_ctx* ctx, int op, const uint8_t* a, const uint8_t* b, size_t n, uint8_t* out)
{
    if (!ctx || !a || !b || !out || op < 0 || op >= FOP_COUNT) return FABGPU_E_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    Device& dv = ctx->devs[0];
    CK(ctx, cudaSetDevice(dv.id));
    DevArray<uint8_t> da, db, dout;
    Grow grow{ctx};
    grow(da, 32 * n); grow(db, 32 * n); grow(dout, 32 * n);
    if (grow.rc) return grow.rc;
    CK(ctx, cudaMemcpy(da.get(), a, 32 * n, cudaMemcpyHostToDevice));
    CK(ctx, cudaMemcpy(db.get(), b, 32 * n, cudaMemcpyHostToDevice));
    fieldop_kernel<<<(unsigned)((n + 63) / 64), 64>>>(op, da.get(), db.get(), (int)n, dout.get());
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dout.get(), 32 * n, cudaMemcpyDeviceToHost));
    return FABGPU_OK;
}

int fabgpu_test_couch_values(fabgpu_ctx* ctx, const uint8_t* blob, const uint32_t* off, size_t n, int path, uint32_t* out)
{
    if (!ctx || (n && (!blob || !off || !out)) || n > UINT32_MAX || path < 0 || path > 2) return FABGPU_E_ARG;
    for (size_t i = 0; i < n; i++) if (off[i + 1] < off[i]) { ctx->last_error = "decreasing offsets"; return FABGPU_E_ARG; }
    if (n == 0) return FABGPU_OK;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(ctx, cudaSetDevice(ctx->devs[0].id));
    const size_t bytes = std::max<size_t>(off[n], 1);
    DevArray<uint8_t> d_b; DevArray<uint32_t> d_o, d_out;
    Grow grow{ctx};
    grow(d_b, bytes); grow(d_o, 4 * (n + 1)); grow(d_out, 4 * n);
    if (grow.rc) return grow.rc;
    CK(ctx, cudaMemcpy(d_b.get(), blob, off[n], cudaMemcpyHostToDevice));
    CK(ctx, cudaMemcpy(d_o.get(), off, 4 * (n + 1), cudaMemcpyHostToDevice));
    bdev::cv_test_kernel<<<(unsigned)((n + 127) / 128), 128>>>(d_b.get(), d_o.get(), (uint32_t)n, path, d_out.get());
    bdev::cv_test_long_kernel<<<(unsigned)std::min<size_t>(n, 1024), bdev::CV_LT_THREADS>>>(d_b.get(), d_o.get(), (uint32_t)n, path, d_out.get());
    ctx->launches += 2;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, d_out.get(), 4 * n, cudaMemcpyDeviceToHost));
    return FABGPU_OK;
}

int fabgpu_test_table_entries(fabgpu_ctx* ctx, int key_slot, const uint32_t* window, const uint32_t* digit, size_t n, uint8_t* out)
{
    if (!ctx || !window || !digit || !out || key_slot >= ctx->kt->key_slots) return FABGPU_E_ARG;
    std::shared_lock<std::shared_mutex> rl(ctx->kt->tab_mu);    // no context of the group recycles a slot, nor enqueues a build, until the copy-back
    std::lock_guard<std::mutex> lk(ctx->mu);
    Device& dv = ctx->devs[0];
    const aff* tab;
    int windows;
    uint32_t stride, dmax;                              // entries per window, largest digit
    if (key_slot <= -2) {
        const int32_t code = handle_to_slot(ctx, key_slot);
        if (code == -1) return FABGPU_E_ARG;            // stale handle, or the slot is no longer in use
        tab = dv.tab->stab.get() + (size_t)(-2 - code) * FAB_S_POINTS;
        windows = FAB_S_WINDOWS; stride = dmax = FAB_S_HALF;
    } else if (key_slot == -1) {
        tab = dv.tab->gtab.get(); windows = FAB_G_WINDOWS; stride = dmax = FAB_G_ENTRIES;
    } else {
        tab = dv.tab->qtab.get() + (size_t)key_slot * FAB_Q_WINDOWS * FAB_Q_ENTRIES; windows = FAB_Q_WINDOWS; stride = dmax = FAB_Q_ENTRIES;
    }
    for (size_t i = 0; i < n; i++)
        if (window[i] >= (uint32_t)windows || digit[i] == 0 || digit[i] > dmax) return FABGPU_E_ARG;
    if (n == 0) return FABGPU_OK;
    CK(ctx, cudaSetDevice(dv.id));
    DevArray<uint32_t> d_w, d_d; DevArray<aff> d_out;
    Grow grow{ctx};
    grow(d_w, 4 * n); grow(d_d, 4 * n); grow(d_out, sizeof(aff) * n);
    if (grow.rc) return grow.rc;
    CK(ctx, cudaMemcpy(d_w.get(), window, 4 * n, cudaMemcpyHostToDevice));
    CK(ctx, cudaMemcpy(d_d.get(), digit, 4 * n, cudaMemcpyHostToDevice));
    // small tables are built on s_stream, which the legacy stream does not wait for: read only after the last build
    if (dv.tab->s_ev_set) CK(ctx, cudaStreamWaitEvent(0, dv.tab->s_ev.get(), 0));
    table_entries_kernel<<<(unsigned)((n + 127) / 128), 128>>>(tab, stride, d_w.get(), d_d.get(), (uint32_t)n, d_out.get());
    ctx->launches++;
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, d_out.get(), sizeof(aff) * n, cudaMemcpyDeviceToHost));
    return FABGPU_OK;
}

}  // extern "C"
