/* fabgpu_ecdsa.h -- C ABI of the H100 batch ECDSA-P256 verifier (libfabgpu_ecdsa.so).
 *
 * Drop-in boundary for ONE path of trustbloc/fabric-mod: signature verification behind
 *     bccsp.BCCSP.Verify(k, signature, digest, opts) (bool, error)         reference bccsp/bccsp.go:123-125
 * as implemented by the software provider
 *     sw.CSP.Verify -> verifyECDSA -> crypto/ecdsa.Verify                   reference bccsp/sw/impl.go:247-270,
 *                                                                           bccsp/sw/ecdsa.go:41-57
 * and reached from msp identity.Verify (reference msp/identities.go:169-196).  The reference has no native
 * code on this path; these entry points are what a cgo provider (INTEGRATION.md, go/bccsp/gpu) binds, in the
 * same way bccsp/pkcs11 binds an HSM library (reference bccsp/pkcs11/pkcs11.go:36-87,241-262).
 *
 * Conventions
 *   - plain pointers and sizes only; no CUDA or torch types.  `cuda_stream` arguments are a cudaStream_t
 *     passed as void* (NULL = CUDA's default stream, as in the runtime API).
 *   - every function returns FABGPU_OK (0) or a negative FABGPU_E_* code.  A negative code means "could not
 *     decide": the caller MUST fall back to the CPU provider for that batch.  A device fault is never
 *     reported as "signature invalid" (SURVEY.md section 5: that would fork the ledger).
 *   - big integers cross the boundary as 32-byte big-endian strings, structure-of-arrays: element i of an
 *     array lives at bytes [32*i, 32*i+32).
 *   - validity bitmask: signature i -> bit (i % 32) of uint32 word (i / 32); 1 = VALID, i.e. (true, nil).
 *   - there is NO CPU fallback inside this library: without a usable CUDA device fabgpu_init fails.
 */
#ifndef FABGPU_ECDSA_H
#define FABGPU_ECDSA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fabgpu_ctx fabgpu_ctx;

enum {
    FABGPU_OK = 0,
    FABGPU_E_NO_DEVICE = -1,   /* no CUDA device / driver, or device id out of range */
    FABGPU_E_CUDA = -2,        /* a CUDA call failed; see fabgpu_last_error */
    FABGPU_E_ARG = -3,         /* bad argument (NULL, n > max_batch, bad slot ...) */
    FABGPU_E_INJECTED = -4     /* FABGPU_FAULT_INJECT=1 is set: every verify call fails (fault-injection tests) */
};

/* Per-signature status of the bccsp-level entry points: the (bool, error) pair of sw.CSP.Verify as one byte.
 * Error kinds follow reference bccsp/sw/impl.go:249-266, bccsp/sw/ecdsa.go:42-54, bccsp/utils/ecdsa.go:43-92. */
enum {
    FABGPU_ST_VALID = 0,              /* (true,  nil) */
    FABGPU_ST_INVALID = 1,            /* (false, nil): well-formed but wrong, incl. r >= N, point at infinity */
    FABGPU_ST_ERR_NIL_KEY = 2,        /* "Invalid Key. It must not be nil." */
    FABGPU_ST_ERR_EMPTY_SIG = 3,      /* "Invalid signature. Cannot be empty." */
    FABGPU_ST_ERR_EMPTY_DIGEST = 4,   /* "Invalid digest. Cannot be empty." */
    FABGPU_ST_ERR_UNMARSHAL = 5,      /* "Failed unmashalling signature [...]" (asn1) */
    FABGPU_ST_ERR_R_NOT_POSITIVE = 6, /* "invalid signature, R must be larger than zero" */
    FABGPU_ST_ERR_S_NOT_POSITIVE = 7, /* "invalid signature, S must be larger than zero" */
    FABGPU_ST_ERR_HIGH_S = 8,         /* "Invalid S. Must be smaller than half the order [..][..]." */
    FABGPU_ST_ERR_UNSUPPORTED_KEY = 9,/* not a P-256 key: delegate to the embedded sw provider */
    FABGPU_ST_ERR_OFF_CURVE = 10      /* public key is not a curve point: outside the reference's defined behaviour, delegate to CPU */
};

/* ---- lifetime ---------------------------------------------------------------------------------------- */

/* Creates a context on the given CUDA devices (device_ids == NULL && n_dev == 0: device 0).  Allocates, per
 * device, the fixed-base table, device SoA buffers and pinned host SoA buffers for `max_batch` signatures per
 * slot (FABGPU_SLOTS slots), and builds the table on the device.  A batch given to the host-buffer entry points
 * is split into contiguous, 32-aligned ranges across the context's devices. */
int fabgpu_init(const int* device_ids, int n_dev, size_t max_batch, fabgpu_ctx** out);
/* Creates a context on `with`'s devices that shares `with`'s point tables and key caches: one context per channel of a peer, all in
 * one GROUP, without a second copy of any table.  The group shares the generator's fixed-base table, the window-table pool (key -> slot
 * map, LRU order, generations, the per-key signature counts that earn tables) and the small-table pool, with the capacities and the
 * FABGPU_KEY_MIN_USES / FABGPU_SMALL_MIN_USES settings read when the group's first context was made; nothing is built here.  The new
 * context owns, exactly as one from fabgpu_init does: its slots, streams, pinned and device batch buffers, gate and block buffers, the
 * MSP view and every policy table, the capability, the tx-id set, the state table and state-database kind, the peer-exchange state,
 * its last error, its launch count and its FABGPU_CACHED_KERNEL choice.
 *   - handles from fabgpu_keys_register{,_small} are valid in every context of the group; a stale handle still costs speed, never
 *     correctness.
 *   - fabgpu_key_slot_capacity, fabgpu_small_slot_capacity and fabgpu_key_table_stats report the group's pools, and fabgpu_msp_configure
 *     compares an MSP's size against the group's window-table capacity.
 *   - recycling is least-recently-used across the group: a registration in one context may recycle a table another context's MSP or
 *     batch uses, and that context registers the key again on its next block (as it does after a recycling in its own context).
 *     Size FABGPU_KEY_SLOTS for the busy endorsers of all channels together.
 *   - with == NULL: FABGPU_E_ARG and *out = NULL.  max_batch follows fabgpu_init's rules.  `with` may itself have been made by this
 *     call: the new context joins the same group.  Contexts of a group may be destroyed in any order; the shared tables go with the
 *     last of them. */
int fabgpu_init_shared(fabgpu_ctx* with, size_t max_batch, fabgpu_ctx** out);
void fabgpu_destroy(fabgpu_ctx* ctx);
/* Last error text of this context (or of the failed fabgpu_init when ctx == NULL). Never NULL. */
const char* fabgpu_last_error(const fabgpu_ctx* ctx);
int fabgpu_device_count(const fabgpu_ctx* ctx);
size_t fabgpu_max_batch(const fabgpu_ctx* ctx);

#define FABGPU_SLOTS 3

/* ---- leaf: pre-gated SoA tuples -> bitmask (replaces the crypto/ecdsa.Verify call at bccsp/sw/ecdsa.go:56) */

/* Pinned, library-owned host SoA buffers of one slot (cgo cannot hand Go memory to an async copy).  Each of
 * qx,qy,e,r,s has max_batch*32 bytes; mask and offcurve have ceil(max_batch/32) words.  Caller pre-conditions,
 * established by the host gates exactly as the reference does before calling ecdsa.Verify: 0 < r, 0 < s <= N/2,
 * r < 2^256 (longer r is INVALID without asking the GPU), e = leftmost min(len,32) digest bytes left-padded. */
int fabgpu_host_buffers(fabgpu_ctx* ctx, int slot, uint8_t** qx, uint8_t** qy, uint8_t** e, uint8_t** r,
                        uint8_t** s, uint32_t** mask, uint32_t** offcurve);
/* H2D + kernel + D2H for the first n tuples of the slot's pinned buffers; synchronous. */
int fabgpu_verify_p256(fabgpu_ctx* ctx, int slot, size_t n);
/* Same, asynchronous: returns after enqueueing; fabgpu_wait blocks until the slot's mask is complete. */
int fabgpu_verify_p256_async(fabgpu_ctx* ctx, int slot, size_t n);
int fabgpu_wait(fabgpu_ctx* ctx, int slot);
/* Convenience for callers whose tuples sit in ordinary host memory: copies through slot 0. */
int fabgpu_verify_p256_host(fabgpu_ctx* ctx, const uint8_t* qx, const uint8_t* qy, const uint8_t* e,
                            const uint8_t* r, const uint8_t* s, size_t n, uint32_t* mask, uint32_t* offcurve);
/* Inputs and outputs already resident in the memory of context device `dev_index`; enqueues on `cuda_stream`
 * and returns without synchronising.  offcurve may be NULL. */
int fabgpu_verify_p256_device(fabgpu_ctx* ctx, int dev_index, const void* d_qx, const void* d_qy, const void* d_e,
                              const void* d_r, const void* d_s, size_t n, void* d_mask, void* d_offcurve,
                              void* cuda_stream);

/* ---- per-key fixed-base tables (SURVEY.md section 8f rank 4; what KeyImport does once per identity) -----------
 * Identities repeat heavily in Fabric (the reference caches them: msp/cache/cache.go:38-129; keys are imported once,
 * bccsp/sw/keyimport.go:114-134, msp/mspimpl.go:420).  A registered key gets a window table on every device of the
 * context, after which u2*Q is fixed-base like u1*G.  Results are identical to the generic kernel; only speed differs. */

/* Looks up / builds tables for K keys (X||Y, 64 bytes each).  slots_out[k] >= 0 is the key's HANDLE
 * ((generation << 12) | slot); -1 means "no table" (not a curve point, or more distinct keys than
 * fabgpu_key_slot_capacity in one call) -- such signatures simply take the generic kernel.  Least-recently-used slots are
 * recycled; a handle issued before its slot was recycled is detected by the pinned-slot entry points and treated as -1,
 * so a stale handle costs speed, never correctness.  Capacity: env FABGPU_KEY_SLOTS (default 256, at most 4096). */
int fabgpu_keys_register(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, int32_t* slots_out);
int fabgpu_key_slot_capacity(const fabgpu_ctx* ctx);
/* The tier between "never seen" and a window table: a SMALL table (33 windows of signed 8-bit digits, 264 KiB, built in
 * about 1.5 us of GPU time) makes u2*Q 33 mixed additions and no doublings.  Meant for keys that recur without being busy -- client /
 * creator certificates, thousands of identities with a few signatures per block each (the reference caches exactly those identities:
 * msp/cache/cache.go:38-129).  handles_out[k] <= -2 is the key's small HANDLE (-2 - ((generation << 20) | slot)), -1 = no slot could
 * be had; every entry point that takes key handles accepts both kinds.  A key that is not a curve point still gets a handle: its
 * signatures are reported off-curve, exactly as by the generic kernel.  The build is enqueued, not waited for; consumers are ordered
 * behind it on the device.  fabgpu_bccsp_verify_batch* give a key a small table by themselves once FABGPU_SMALL_MIN_USES (default 32: the
 * point where the key has cost as much on the generic kernel as its table does) of its signatures have been seen without a window table; fabgpu_msp_configure uses small tables when the MSP holds more identities
 * than window-table slots.  Capacity: env FABGPU_SMALL_SLOTS (default 16 384 = 4.4 GB per device; 0 turns the tier off); least recently
 * used tables are recycled in bulk (stale handles are detected like the big ones). */
int fabgpu_keys_register_small(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, int32_t* handles_out);
int fabgpu_small_slot_capacity(const fabgpu_ctx* ctx);
/* Build constants of the small tables: signed window width in bits, number of windows, bytes per table. */
void fabgpu_small_table_info(int* window_bits, int* windows, size_t* table_bytes);
/* out[0] = window tables alive, out[1] = small tables alive, out[2] = small tables built so far, out[3] = small tables recycled. */
int fabgpu_key_table_stats(fabgpu_ctx* ctx, unsigned long long out[4]);
/* Pinned int32[max_batch] of one slot: key_slot[i] = handle of signature i's key (from fabgpu_keys_register), or -1.
 * Only the _keyed entry points read it (they replace handles by live slot indices in place); callers overwrite all n
 * entries per batch and still fill Qx/Qy, which the generic kernel uses whenever a handle is -1 or stale. */
int fabgpu_host_key_slots(fabgpu_ctx* ctx, int slot, int32_t** key_slot);
int fabgpu_verify_p256_keyed(fabgpu_ctx* ctx, int slot, size_t n);
int fabgpu_verify_p256_keyed_async(fabgpu_ctx* ctx, int slot, size_t n);
/* Device-resident form: d_key_slot holds raw slot indices (handle & 0xfff) that the caller obtained from
 * fabgpu_keys_register and knows to be live: RAW slots are not re-validated, so the caller must not let a registration that could
 * recycle them (fabgpu_keys_register of new keys, fabgpu_msp_configure, a fabgpu_bccsp_verify_batch* call that tables new keys) run
 * between obtaining the slots and the completion of this launch.  The handle-taking entry points (fabgpu_verify_p256_keyed*,
 * fabgpu_bccsp_verify_batch*, fabgpu_validate_*) hold the library's slot-table lock from resolution to enqueue and need no such care.
 * all_cached = 1 promises every d_key_slot[i] >= 0 (d_qx/d_qy may then be NULL); all_cached = 2 promises every d_key_slot[i] <= -2,
 * the raw code of a small table: -2 - (slot bits of a small handle, i.e. (-2 - handle) & 0xfffff); all_cached = 0: any mix (this form has
 * no compaction scratch: every signature without a WINDOW table -- codes -1 and <= -2 alike -- goes through the generic arithmetic
 * and reads d_qx/d_qy). */
int fabgpu_verify_p256_device_keyed(fabgpu_ctx* ctx, int dev_index, int all_cached, const void* d_key_slot, const void* d_qx,
                                    const void* d_qy, const void* d_e, const void* d_r, const void* d_s, size_t n,
                                    void* d_mask, void* d_offcurve, void* cuda_stream);

/* ---- validity bitmask across GPUs driven by separate processes (one process per GPU, SURVEY.md section 8e) ----------------
 * The reference has no counterpart (its verifier is per-signature, bccsp/sw/ecdsa.go:41-57); BASELINE.json's north_star asks for
 * the batch to be split across the GPUs of a box and the bitmask to be reassembled.  The consumer of the bitmask is the HOST
 * (the Go provider reads it from pinned memory), so the single-process form (one context, several devices: fabgpu_verify_p256*)
 * needs no device-to-device collective at all.  For the one-process-per-GPU form the library exchanges the mask words itself,
 * over peer memory: every rank creates a receive buffer and exports it (CUDA IPC), maps the others', and the verify kernel's
 * epilogue stores each ballot word into the buffer of every rank (P2P writes over NVLink / NVSwitch), followed by a step flag;
 * a wait kernel on the same stream returns when all ranks' words of that step have landed.  No NCCL call on the data path
 * (fabric-mod_b200/sharding.py keeps the NCCL all-gather as the alternative).
 *   _create: this rank's buffer for `world` ranks x words_per_rank mask words; writes its IPC handle (FABGPU_IPC_HANDLE_BYTES).
 *   _open:   handles = world x FABGPU_IPC_HANDLE_BYTES bytes, rank-major (the caller exchanges them, e.g. over its process group).
 *   _allgather: fabgpu_verify_p256_device_keyed for this rank's n signatures (n <= 32 x words_per_rank), then the exchange;
 *            `step` must be 1, 2, 3, ... in lock step on all ranks; *d_full_mask = device pointer to world x words_per_rank
 *            words, valid once the stream has run (until step + 2 is launched: two generations).  A peer that never publishes
 *            makes the NEXT call fail with FABGPU_E_CUDA instead of hanging the GPU. */
#define FABGPU_IPC_HANDLE_BYTES 64
int fabgpu_peer_mask_create(fabgpu_ctx* ctx, int dev_index, int world, int rank, size_t words_per_rank,
                            uint8_t handle_out[FABGPU_IPC_HANDLE_BYTES]);
int fabgpu_peer_mask_open(fabgpu_ctx* ctx, int dev_index, const uint8_t* handles);
int fabgpu_peer_mask_close(fabgpu_ctx* ctx, int dev_index);
int fabgpu_verify_p256_device_keyed_allgather(fabgpu_ctx* ctx, int dev_index, int all_cached, const void* d_key_slot,
                                              const void* d_qx, const void* d_qy, const void* d_e, const void* d_r,
                                              const void* d_s, size_t n, uint32_t step, void** d_full_mask, void* cuda_stream);

/* ---- bccsp level: raw DER signatures + digests + keys -> three-valued status (sw.CSP.Verify semantics) -- */

/* keys_xy: K x 64 bytes (X || Y, big-endian).  key_idx[i] in [0,K), or < 0 for a nil key.  digests / sigs are
 * concatenations indexed by (n+1)-entry offset tables.  status[i] receives FABGPU_ST_*.  The gates (DER per Go
 * encoding/asn1, positivity, low-S, r < 2^256) run in a kernel in front of the verify kernel (on the context's host
 * threads for multi-device contexts or with FABGPU_BCCSP_HOST_GATES=1); survivors are verified.  Keys used by at least
 * FABGPU_KEY_MIN_USES (env, default 256; negative disables) signatures of the call get a window table automatically.
 * A call of >= 24576 signatures is cut into one chunk per slot internally when all slots are free. */
int fabgpu_bccsp_verify_batch(fabgpu_ctx* ctx, const uint8_t* keys_xy, int K, const int32_t* key_idx,
                              const uint8_t* digests, const uint32_t* dig_off, const uint8_t* sigs,
                              const uint32_t* sig_off, size_t n, uint8_t* status);
/* The same call in two halves, for a caller that keeps the GPU fed (the Go provider's aggregator): _async stages the
 * batch into the slot's pinned buffers and enqueues copies + kernels + the status read-back on the slot's stream, then
 * returns -- the caller's arrays are not referenced afterwards; _wait blocks until that batch is done and writes its n
 * status bytes.  With the FABGPU_SLOTS slots used round-robin, the staging and copies of the next batches overlap the kernels of batch i.
 * A slot holds one batch at a time (FABGPU_E_ARG otherwise); fabgpu_bccsp_verify_batch itself is _async + _wait on slot 0. */
int fabgpu_bccsp_verify_batch_async(fabgpu_ctx* ctx, int slot, const uint8_t* keys_xy, int K, const int32_t* key_idx,
                                    const uint8_t* digests, const uint32_t* dig_off, const uint8_t* sigs,
                                    const uint32_t* sig_off, size_t n);
int fabgpu_bccsp_verify_batch_wait(fabgpu_ctx* ctx, int slot, uint8_t* status, size_t n);
/* Zero-copy form of the pair above (what the Go provider's block pre-pass and bench.py's e2e leg use): the library hands out
 * the slot's PINNED staging buffers, the caller writes the batch there -- keys (K x 64 B), key index per signature, digest and
 * DER blobs with their offset tables (offsets start at 0) -- and _inplace_async enqueues the copies and kernels straight from
 * them; no second host copy, no staging threads.  The buffers stay valid (and keep their contents) until a later
 * fabgpu_bccsp_batch_buffers call asks for larger capacities; they must not be rewritten while the slot's batch is in flight.
 * Single-device contexts; completion and statuses through fabgpu_bccsp_verify_batch_wait. */
int fabgpu_bccsp_batch_buffers(fabgpu_ctx* ctx, int slot, size_t n_cap, size_t sig_bytes_cap, size_t dig_bytes_cap, int k_cap,
                               uint8_t** keys_xy, int32_t** key_idx, uint8_t** digests, uint32_t** dig_off, uint8_t** sigs,
                               uint32_t** sig_off);
int fabgpu_bccsp_verify_batch_inplace_async(fabgpu_ctx* ctx, int slot, int K, size_t n);
/* Single call with the reference's exact error strings (sw.CSP.Verify).  key_xy == NULL is the nil key.
 * *valid and err (NUL-terminated, truncated to errcap) mirror the Go (bool, error) pair; err[0] == 0 is nil. */
int fabgpu_bccsp_verify(fabgpu_ctx* ctx, const uint8_t* key_xy, const uint8_t* sig, size_t sig_len,
                        const uint8_t* digest, size_t digest_len, int* valid, char* err, size_t errcap);
/* The host gate alone (no GPU): parses one DER signature the way utils.UnmarshalECDSASignature + IsLowS do and,
 * on success, writes r and s as 32-byte big-endian.  Returns a FABGPU_ST_* code: FABGPU_ST_VALID means "gates
 * passed, ask the GPU"; FABGPU_ST_INVALID means r >= 2^256 (cannot be < N). */
int fabgpu_gate_signature(const uint8_t* sig, size_t sig_len, uint8_t r_out[32], uint8_t s_out[32]);

/* ---- block level: the signature pre-pass of TxValidator.Validate (SURVEY.md section 8a rows a11-a14, 8f ranks 1-2) ----
 * One call verifies every signature of a serialized common.Block as ONE GPU batch -- creator signatures
 * (core/common/validation/msgvalidation.go:26-64) and endorsement signatures (statebased/validator_keylevel.go:243-259,
 * common/policies/policy.go:365-402) -- with the SHA-256 of each signed message computed on the device straight from the
 * block bytes, then replays the reference's per-transaction decision order (msgvalidation.go:248-320, v20/validator.go:
 * 300-455, cauthdsl.go:24-92, markTXIdDuplicates) and writes the TRANSACTIONS_FILTER bytes (peer.TxValidationCode).
 * The ledger's inputs come as tables the caller installs: chaincode definitions (_namespace_policies, _namespace_versions), collection
 * and key-level policies, and the committed tx ids (fabgpu_committed_txids): once a set is installed, a transaction whose id the ledger
 * already holds is DUPLICATE_TXID (9) as in the reference; without one the device does not look ids up in the ledger.  Config
 * transactions are flagged 254 (NOT_VALIDATED) and must be validated by the CPU validator. */

/* Installs the MSP view and the endorsement policy used by fabgpu_validate_block.
 * identities: n_ids serialized msp.SerializedIdentity byte strings (id_blob + (n_ids+1) offsets) exactly as they appear in
 * SignatureHeader.creator / Endorsement.endorser, their MSP ids, P-256 keys (X||Y) and the outcome of identity.Validate().
 * policy_nodes: n_nodes x 4 int32 (type, n, first_child, n_children); type 0 = NOutOf(n) over children
 * [first_child, first_child + n_children), type 1 = SignedBy(principal n), type 2 = ImplicitMeta with threshold n over the
 * children (common/policies/implicitmeta.go:44-103: satisfied iff at least n children are, each child evaluated as a policy of
 * its own, so one signer may satisfy several); node 0 is the root.  Principals are named by strings.  By default a principal
 * is an MSP id matched as ROLE MEMBER: a signer satisfies it iff its MSP id is that string and its Validate() passed.
 * fabgpu_msp_principal_bits replaces that match by the caller's own SatisfiesPrincipal answers (roles, identities, OUs).
 * Every identity's key gets a window table when the MSP fits the window-table pool (n_ids <= fabgpu_key_slot_capacity);
 * a larger MSP -- thousands of client certificates -- goes to the small tier instead, except the identities whose key already owns a
 * window table: register the few busy keys (the endorsing peers) with fabgpu_keys_register BEFORE this call and they keep it.
 * FABGPU_E_ARG, with nothing installed, for a policy array the device cannot evaluate exactly: a node type other than 0, 1
 * or 2, children outside the array, a SignedBy index outside the principals, an ImplicitMeta node below an NOutOf node or
 * with a threshold outside [1, n_children] (0 is accepted only with no children), a cycle, or a tree deeper than 12 levels
 * below any node (BD_MAX_POLICY_DEPTH; ImplicitMeta nodes count as levels).  The caller then validates that channel's blocks
 * on the CPU. */
int fabgpu_msp_configure(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob,
                         const uint32_t* mspid_off, const uint8_t* keys_xy, const uint8_t* valid, int n_ids,
                         const int32_t* policy_nodes, int n_nodes, const uint8_t* principal_blob, const uint32_t* principal_off,
                         int n_principals, const char* channel_id);
/* Optional refinements of the table fabgpu_msp_configure installed (call them after it; each drains the block slots first;
 * fabgpu_msp_configure clears all four -- but not the committed tx-id set, which is ledger state, not channel configuration):
 *   _identity_groups: group[i] = de-duplication id of identity i.  The reference de-duplicates a transaction's signers on
 *       Mspid + certificate digest (common/policies/policy.go:380-386), so two byte-different serializations of ONE certificate
 *       must share a group; without this call every table entry is its own group.
 *   _namespace_policies: the endorsement policy of each chaincode namespace (what the plugin dispatcher looks up per namespace a
 *       transaction writes to, core/committer/txvalidator/v20/plugindispatcher/dispatcher.go:166-221,265-277): ns_root[i] is the
 *       root node -- an index into the node array given to fabgpu_msp_configure, which may hold several trees -- of namespace i's
 *       policy.  n_ns = 0 restores "node 0 is the policy of every namespace".  A transaction that needs a namespace without an
 *       entry is flagged 254 (NOT_VALIDATED): the CPU validator reads the chaincode definition from the ledger.
 *   _principal_bits: which identity satisfies which principal, W = ceil(n_principals / 32) words per identity: bit p % 32 of
 *       bits[i * W + p / 32] set iff identity i satisfies principal p -- the caller's msp Identity.SatisfiesPrincipal(principal)
 *       == nil, so MSP version, NodeOUs, admin lists, IDENTITY and ORGANIZATION_UNIT principals are answered where the
 *       reference answers them (msp/mspimpl.go); the device never parses certificates.  While bits are installed, SignedBy(p)
 *       matches a verified, de-duplicated signer iff its bit p is set, whatever its Validate() outcome (an admin-listed
 *       identity satisfies ADMIN without it, mspimpl.go:506-513); the creator's Validate() is still checked.  n_ids and
 *       n_principals must equal fabgpu_msp_configure's, else FABGPU_E_ARG and nothing changes; n_ids = 0 removes the bits
 *       and restores MSP-id member matching.
 *   (_identity_groups and _principal_bits take the identities the table holds now: those fabgpu_msp_configure installed, then those
 *       fabgpu_msp_identities_add admitted, in that order.)
 *   _collection_policies: the endorsement policy of private-data collections.  Entry i says that a write to collection coll[i]
 *       (coll_blob + (n+1) offsets) of namespace ns[i] (ns_blob + (n+1) offsets) is checked against the tree at node coll_root[i] of
 *       fabgpu_msp_configure's array instead of the chaincode's (core/common/validation/statebased/v20.go:105-147).  The caller
 *       resolves CollectionValidationInfo (core/chaincode/lifecycle/deployedcc_infoprovider.go:359-394): an implicit
 *       collection _implicit_org_<MSPID> gets that org's Endorsement policy, or SignedByAnyMember(MSPID) without one; a static
 *       collection with an EndorsementPolicy gets it; one without gets its chaincode's root.  While a table is installed, each
 *       validated namespace must satisfy the policy of every named collection it writes (hashed writes or hashed metadata
 *       writes), its chaincode policy when it has public writes or writes to a collection without a name, and its chaincode
 *       policy when it wrote nothing else.  A transaction that writes a (namespace, collection) without an entry, or more than
 *       8 named collections, is flagged 254 (NOT_VALIDATED).  FABGPU_E_ARG, with the previous table kept, for NULL arrays with
 *       n > 0, a root outside [0, n_nodes), decreasing offsets, an empty collection name or a (namespace, collection) given twice.
 *       n = 0 removes the table: every write falls under its namespace's chaincode policy, as without this call. */
int fabgpu_msp_identity_groups(fabgpu_ctx* ctx, const int32_t* group, int n_ids);
int fabgpu_msp_principal_bits(fabgpu_ctx* ctx, const uint32_t* bits, int n_ids, int n_principals);
/* Identity admission: appends n identities to the table fabgpu_msp_configure installed, in its encoding (serialized bytes, MSP id,
 * X||Y, Validate() outcome), without draining the block slots -- the table the device reads while blocks are in flight.  A new MSP id
 * gets a code of its own, which matches no principal of the policies.  group: one de-duplication id per identity (it may name an
 * existing group, e.g. another serialization of a held certificate), given iff a group table is installed; bits: W words per identity
 * (W of fabgpu_msp_principal_bits), given iff principal bits are installed.  Ordering as for fabgpu_committed_txids_add: blocks submitted
 * before the call returns never see the new identities, every block submitted after it does; the host never waits for blocks in
 * flight.  Each admitted key gets a small table (or keeps the window table it owns); with no small slot free it goes through the
 * generic kernel.  FABGPU_E_ARG, with nothing enqueued and the table unchanged, for: no configured table, n < 0, NULL arrays with
 * n > 0, decreasing offsets, an empty identity, an identity the table holds (equal bytes) or one given twice, group or bits present
 * when it must be absent or absent when it must be present, a negative group.  fabgpu_msp_configure replaces admitted identities
 * too.  Contexts of one table group (fabgpu_init_shared) admit independently. */
int fabgpu_msp_identities_add(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob, const uint32_t* mspid_off,
                              const uint8_t* keys_xy, const uint8_t* valid, const int32_t* group, const uint32_t* bits, int n);
int fabgpu_namespace_policies(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const int32_t* ns_root, int n_ns);
int fabgpu_collection_policies(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob,
                               const uint32_t* coll_off, const int32_t* coll_root, int n);
/* Key-level endorsement policies (state-based endorsement; core/common/validation/statebased/validator_keylevel.go:37-142,
 * vpmanagerimpl.go:196-362).  Also a refinement: it drains the block slots, and fabgpu_msp_configure clears it.
 *   _key_policies replaces the table.  Entry i maps (namespace ns[i], collection coll[i], key key[i]) -- three blobs with (n+1)
 *       offsets each; the collection is empty for a public key, and for a private-data key the key is its 32-byte key hash -- to
 *       the validation parameter compiled to `nodes` (n_nodes x 4 ints in fabgpu_msp_configure's format, NOutOf and SignedBy only,
 *       child indices counted within this call's array, SignedBy indexing fabgpu_msp_configure's principals): root[i] is a node of
 *       this call's array, or -2 when the key's parameter is not one the device may decide (it does not translate, or names a
 *       principal outside the configured list); a transaction writing such a key is flagged 254.  The library appends the nodes
 *       after the configured ones.  n = 0 with n_nodes = 0 removes the table.
 *   _key_policies_update upserts entries into the installed table with the same arguments; root -1 removes an entry (removing an
 *       absent key does nothing).  Its cost follows the size of the change, not of the table: what a peer calls after committing
 *       each block, with the validation parameters that block's valid metadata writes set or cleared.
 *   While a table is installed, each write of a validated namespace -- public write, public metadata write, hashed write, hashed
 *   metadata write -- is checked against its key's entry if it has one and then not against its chaincode or collection policy;
 *   otherwise against its collection's policy (with a collection table; a written collection without an entry is flagged 254) or
 *   its chaincode's.  A validated namespace without writes is checked against its chaincode policy.  More than 16 distinct
 *   policies for one transaction is flagged 254.  A transaction that writes a key some earlier transaction of the block
 *   metadata-wrote waits for that transaction's result: ENDORSEMENT_POLICY_FAILURE (10) if it was VALID, its own flag if it failed
 *   its policy for its only namespace, and 254 in every other case (the reference would wait for a result that never comes).
 *   Both calls return FABGPU_E_ARG with a fabgpu_last_error text, and keep the previous table, for NULL arrays with n > 0,
 *   decreasing offsets, a node type other than 0 or 1, a child or root out of range, a cycle, a tree deeper than 12, a principal
 *   out of range, a (namespace, collection, key) given twice, -1 in a replacing call, and an update with no table installed. */
int fabgpu_key_policies(fabgpu_ctx* ctx, const int32_t* nodes, int n_nodes, const uint8_t* ns_blob, const uint32_t* ns_off,
                        const uint8_t* coll_blob, const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off,
                        const int32_t* root, int n);
int fabgpu_key_policies_update(fabgpu_ctx* ctx, const int32_t* nodes, int n_nodes, const uint8_t* ns_blob, const uint32_t* ns_off,
                               const uint8_t* coll_blob, const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off,
                               const int32_t* root, int n);
/* The channel's validator (core/committer/txvalidator/router.go:43).  Also refinements: each drains the block slots, and
 * fabgpu_msp_configure resets both (back to FABGPU_CAP_V2_0, versions dropped).
 *   _channel_capability: FABGPU_CAP_V2_0 (the default) for a channel whose application capability has V2_0Validation: the v2.0
 *       validator with the plugin dispatcher.  FABGPU_CAP_V1_3 for a V1_3, V1_4_2 or V1_4_3 channel: the v1.4 validator
 *       (core/committer/txvalidator/v14) with the builtin v13 VSCC.  In that mode:
 *       - an empty or mismatched chaincode name, or an empty version, is INVALID_OTHER_REASON (255) instead of 25;
 *       - an application chaincode writing to lscc, vscc, escc or cscc, and an invocation of vscc or escc, is ILLEGAL_WRITESET (23);
 *       - an invocation of qscc or cscc validates only that namespace, against its namespace-table entry (the reference uses
 *         SignedByAnyMember over the channel's MSP ids), without a version check;
 *       - an application chaincode's namespaces are validated in order, the invoked one first, and the first failure decides: a
 *         namespace without a table entry is 254 only when those before it passed;
 *       - the invoked chaincode's version (ChaincodeAction.chaincode_id.version) must equal its lscc version: EXPIRED_CHAINCODE (17)
 *         otherwise, 254 when no version is installed for it;
 *       - each namespace is checked on its own writes: a key's validation parameter if the key table holds one, otherwise the
 *         chaincode policy; the collection policies are not used;
 *       - an invocation of lscc (deploy / upgrade) is 254, and so is every transaction of that block that would be VALID: an
 *         upgrade invalidates the block's later invocations of the chaincode it names, which the device does not decide.  This
 *         holds for every lscc invocation flagged 254, whatever stopped it (a creator outside the table, more than 8 namespaces);
 *         one flagged with another code is one the reference rejects too, and leaves the block's flags alone.
 *       Any other value is FABGPU_E_ARG and the mode is kept.  So is FABGPU_CAP_V1_3 while a namespace root reaches an ImplicitMeta
 *       node: lscc chaincode definitions hold signature policies.  V1_2 and older capabilities are not supported.
 *   _namespace_versions: the lscc ChaincodeData.Version of each entry of the installed namespace table (_namespace_policies, in
 *       its order): ver_blob with (n_ns + 1) offsets, an empty string for no version.  n_ns must equal the table's size, else
 *       FABGPU_E_ARG and nothing changes; n_ns = 0 with an empty table drops the versions.  _namespace_policies drops them too.
 *   On a V1_3 channel the namespace table lists the chaincodes whose lscc ChaincodeData.Vscc is "vscc", with the policy of their
 *   ChaincodeData.Policy, plus qscc and cscc with SignedByAnyMember(channel MSP ids); a chaincode with another VSCC is left out,
 *   so its transactions are 254.  While FABGPU_CAP_V1_3 is set, _namespace_policies refuses a root that reaches an ImplicitMeta
 *   node, and an empty table (n_ns = 0) when node 0 -- then every namespace's policy -- reaches one (FABGPU_E_ARG, the previous
 *   table kept). */
enum { FABGPU_CAP_V2_0 = 0, FABGPU_CAP_V1_3 = 1 };
int fabgpu_channel_capability(fabgpu_ctx* ctx, int cap);
int fabgpu_namespace_versions(fabgpu_ctx* ctx, const uint8_t* ver_blob, const uint32_t* ver_off, int n_ns);
/* The ledger's committed transaction ids, for checkTxIdDupsLedger (core/committer/txvalidator/v20/validator.go:363-372,462-491,
 * v14/validator.go:334-345).  Ids are ChannelHeader.tx_id byte strings: id_blob with n + 1 offsets; kind[i] (kind NULL = all 0) says
 * what the ledger's GetTransactionByID answers for id i: 0 = found (the block store indexes the id of every transaction of every
 * committed block, whatever its flag), 1 = indexed but the lookup fails (ids imported from a snapshot, whose index value is empty).
 *   fabgpu_committed_txids replaces the set; n = 0 with capacity_hint = 0 removes it.  capacity_hint (ids) sizes the table up front.
 *       It drains the block slots first.
 *   fabgpu_committed_txids_add upserts ids into the installed set without draining the slots: what a peer calls with a block's ids
 *       right after submitting that block.  FABGPU_E_ARG when no set is installed.
 *   An id given twice keeps the larger kind.  Only canonical ids are kept -- 64 characters of [0-9a-f], stored as 32 binary bytes: a
 *   transaction reaches the ledger check only after CheckTxID has passed, so its id is the lowercase hex of SHA-256(nonce || creator),
 *   and an id in any other form (uppercase, another length, empty) can never match.
 *   Ordering: an add or replace is never seen by a block submitted before the call (its own ids do not flag it), and is seen by every
 *   block submitted after the call returns.  The caller's arrays are not referenced after the call returns.
 *   While a set is installed, an endorser transaction that passed the checks up to TARGET_CHAIN_NOT_FOUND (14) is DUPLICATE_TXID (9)
 *   when its id has kind 0 and 254 when it has kind 1, before the dispatcher, the chaincode definitions and the policies decide
 *   anything, in both validator modes.  A ledger duplicate is not VALID, so it takes no part in the in-block duplicate pass, and a later
 *   writer of a key it metadata-writes is 254.  Config transactions stay 254.
 *   Memory: 36 bytes per slot, a power-of-two slot count at a load of at most 1/2 (at least 1024 slots): 2^25 slots, 1.2 GB, for 10^7
 *   ids.  The table doubles as ids are added; FABGPU_TXID_MAX_BYTES (environment) bounds its bytes.  When growing or inserting fails
 *   (that bound, or an allocation failure) the call returns an error and the set is broken: every transaction that reaches the ledger
 *   check is 254, and _add is refused, until a fabgpu_committed_txids call succeeds.  The device never answers "not found" from a set
 *   that lacks ids.
 *   FABGPU_E_ARG, with a fabgpu_last_error text and the previous set kept, for NULL arrays with n > 0, decreasing offsets and a kind
 *   other than 0 or 1.  fabgpu_msp_configure keeps the set.
 *   fabgpu_committed_txids_info: out[0] = distinct ids held (0 while broken or removed), out[1] = table slots.
 *   fabgpu_committed_txids_add_block upserts, with kind 0, the ids the block store indexes for the block of `slot`: the id
 *       protoutil.GetOrComputeTxIDFromEnvelope gives for every envelope, whatever its flag -- a non-empty ChannelHeader.tx_id (kept only
 *       when canonical), else hex(SHA-256(nonce || creator)) of its SignatureHeader; nothing for an envelope, payload, header or channel
 *       header that does not unmarshal, a payload without a header, or (with an empty tx_id) a signature header that does not.  The ids
 *       are extracted and inserted on the device: the host neither parses the block nor waits.  Call it after
 *       fabgpu_validate_{block,envelopes}_async(slot) (or a blocking fabgpu_validate_block / _envelopes, slot 0) has returned and before
 *       the slot's next submit; ordering is that of _add.  The slot's next submit waits on the device for the add to have read the
 *       slot's block.  FABGPU_E_ARG, nothing enqueued, when no set is installed, the set is broken, the slot holds no submitted block,
 *       or its block was already added.  Growth is decided on the ids held plus those sent since plus the block's transactions. */
int fabgpu_committed_txids(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* kind, size_t n, size_t capacity_hint);
int fabgpu_committed_txids_add(fabgpu_ctx* ctx, const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* kind, size_t n);
int fabgpu_committed_txids_info(const fabgpu_ctx* ctx, unsigned long long out[2]);
int fabgpu_committed_txids_add_block(fabgpu_ctx* ctx, int slot);
/* The ledger's MVCC check (core/ledger/kvledger/txmgmt/validation/validator.go:82-281), an opt-in stage after the validator, over a
 * device-resident table of the world state's committed key versions with LevelDB semantics (CouchDB's key and value checks: see
 * fabgpu_state_database).  Entry i of a call is (namespace, collection, key) -> (ver[2i], ver[2i+1]) = (block_num, tx_num): three blobs with n + 1
 * offsets each; the collection is empty for a public key, and for a private-data key the key is its 32-byte key hash.
 *   fabgpu_state_versions replaces the table; `height` is the ledger height (committed blocks), so the next block to check is block
 *       `height`.  capacity_hint (keys) sizes the table up front.  n = 0 with capacity_hint = 0 removes it.  It drains the block slots.
 *   fabgpu_state_versions_update upserts entries; a version of (UINT64_MAX, UINT64_MAX) removes the key.  height must be >= the table's;
 *       a larger one closes a block the device left open.
 *   fabgpu_state_versions_info: out[0] = keys held (present or unknown), out[1] = table slots, out[2] = height, out[3] = keys unknown;
 *       keys and unknown keys are 0 while broken or removed.
 *   fabgpu_validate_mvcc checks block `block_num` (= the table's height) held by `slot` after fabgpu_validate_wait returned it and before
 *       the slot's next submit.  tv_flags are the validator's n flags (the device's own, or with some 254s settled by the CPU validator);
 *       flags receives the committed ones: a VALID transaction becomes VALID, MVCC_READ_CONFLICT (11) or 254, every other flag is copied.
 *       254 is given to a transaction with a range query while no index is installed (see fabgpu_state_versions_indexed), one that reads a key an undetermined earlier
 *       transaction of the block writes or that the table marks unknown, one after a transaction whose write set cannot be enumerated,
 *       and one whose applyWriteSet would put a nil value, where the reference panics: a write without a value, or the metadata path
 *       (tx_ops.go adds the operations' flags per key, so two writes or two deletes of one key also take it) on a key an earlier
 *       transaction of the block deleted or an undetermined one wrote.
 *       Then the block is applied at (block_num, tx index): the writes of every transaction left VALID; the keys written by a
 *       transaction left at 254 become unknown, and a later read of an unknown key is 254 until _update gives it a version or removes
 *       it.  When some VALID or 254 transaction's write set cannot be enumerated (no ChaincodeAction.results reached, a non-endorser
 *       transaction) the block stays open: the height does not advance, and the next call is refused until
 *       _update(..., height = block_num + 1) supplies those writes.  Otherwise the height becomes block_num + 1.
 *   FABGPU_E_ARG, with a fabgpu_last_error text and nothing changed, for no table installed, block_num other than the height, an open
 *   block, a slot without a finished block, n other than the block's transaction count, NULL arrays with n > 0, decreasing offsets, and
 *   a key given twice in one call.
 *   Memory: 56 bytes per slot, a power-of-two slot count at a load of at most 1/2 (at least 1024 slots).  FABGPU_STATE_MAX_BYTES
 *   (environment) bounds the table; when growing or inserting fails the call returns an error and the table is broken: every VALID
 *   transaction is 254 and nothing is applied, until a fabgpu_state_versions call succeeds.  fabgpu_msp_configure keeps the table.
 *   The table lives on device 0; blocks in flight on other slots never read it. */
int fabgpu_state_versions(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                          const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height, size_t capacity_hint);
int fabgpu_state_versions_update(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                                 const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height);
int fabgpu_state_versions_info(const fabgpu_ctx* ctx, unsigned long long out[4]);
int fabgpu_validate_mvcc(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* tv_flags, uint8_t* flags, size_t n);
/* Range queries (phantom reads) in fabgpu_validate_mvcc, opt-in: an ordered index of the table's public keys (entries with an empty
 * collection), in bytewise (namespace, key) order, each with its key's digest.  The index only says which keys of a range may exist;
 * presence and version always come from the table, so a removed key may stay in the index as a dead entry until the next install.
 *   fabgpu_state_versions_indexed takes fabgpu_state_versions' arguments, replaces the table the same way, and installs the index over
 *       the call's public keys.  A plain fabgpu_state_versions call drops the index; so does a failure that breaks the table.
 *   While an index is installed, fabgpu_state_versions_update and fabgpu_validate_mvcc add to it every public key the table comes to hold
 *       (present, or unknown after a 254 writer) that it lacks; later insertions go to a small sorted delta, folded into the sorted base
 *       once it passes max(4096, min(base / 8, 2^18)) entries.
 *   fabgpu_validate_mvcc then gives a VALID transaction with range queries VALID, 11 or 254 by validateRangeQuery (validator.go:216-237,
 *       LevelDB): the results of [start_key, end_key) -- an empty end_key is the rest of the namespace -- over the committed state and
 *       the writes of the block's earlier VALID transactions (theirs win; a deleted key is skipped; a metadata write on a present key
 *       re-puts it at (block, tx)), and, when itr_exhausted is false, the end key served once after everything else (from those writes,
 *       else from the table, not at all when absent or deleted; also when start_key > end_key or end_key is empty).
 *       raw_reads (or neither oneof field: no reads) must equal the results exactly, key and version, with none left over.
 *       reads_merkle_hashes must equal the summary RangeQueryResultsHelper(max_degree).Done() builds over the results; max_degree or
 *       fewer results give no summary, hence 11.  Results are drawn as the reference's validators draw them, early exits included.
 *       254 where the reference panics: a raw read without a Version reached with a result of its key, and rangeQueryHashValidator's
 *       early-exit loop indexing the top level out of range (the top level rising after its first matched hash).
 *       254 for max_degree < 2 (the reference fails the commit), a result candidate whose state is unknown (the table marks it, or an
 *       undetermined earlier transaction of the block writes it), and a RangeQueryInfo this stage does not decode: one that does not
 *       parse, both oneof fields present, a oneof field repeated, a max_degree or max_level beyond 32 bits.
 *       Without an index every entry point behaves as above, range queries included (254).
 *   fabgpu_state_index_info: out[0] = index entries the table holds (present or unknown), out[1] = entries including dead ones,
 *       out[2] = the index's device bytes; all 0 without an index.
 *   Memory: 48 bytes per entry plus the key bytes, with room for growth; the index counts toward FABGPU_STATE_MAX_BYTES, and a failed
 *   growth or insert breaks the table (and drops the index) as a failed table growth does. */
int fabgpu_state_versions_indexed(fabgpu_ctx* ctx, const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                                  const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t height, size_t capacity_hint);
int fabgpu_state_index_info(const fabgpu_ctx* ctx, unsigned long long out[3]);
/* The state database fabgpu_validate_mvcc restates, a context property: FABGPU_STATEDB_LEVELDB (the default) or FABGPU_STATEDB_COUCHDB;
 * FABGPU_E_ARG for any other kind.  It changes only what later fabgpu_validate_mvcc calls do; fabgpu_state_versions* and
 * fabgpu_msp_configure keep it.  While CouchDB is set:
 *   fabgpu_validate_mvcc first runs validateWriteset (batch_preparer.go:317-330) with CouchDB's ValidateKeyValue (statecouchdb.go:427,
 *       couchdoc_conv.go:37-57,278-297) over every transaction tv_flags leaves VALID and whose write set the stage enumerates: each public
 *       KVWrite's key, and its value when the field is present (a delete's too); hashed and metadata writes are not checked.
 *       A key is invalid when it is empty, starts with '_', or is not valid UTF-8 (utf8.ValidString).  A value is invalid when Go 1.14's
 *       json.Unmarshal into a map[string]interface{} succeeds -- RFC 8259 grammar as encoding/json's scanner reads it, a top-level object
 *       (or null, which has no fields), no number whose float64 overflows -- and a top-level member name, unescaped, is "~version" or
 *       starts with '_'.  A transaction with an invalid write is INVALID_WRITESET (24): it drops out before the MVCC check, its reads
 *       unchecked and its writes neither applied nor made unknown.  Otherwise it is 254 when some write is undecided: a value nested
 *       deeper than 128 containers, or one holding a reserved name
 *       and a number within the 40 leading digits of the overflow bound or with an exponent of 10000 or more.  It is also 254 when it
 *       reads a public key CouchDB cannot hold, has a range whose start or end key is not UTF-8, or has a range with itr_exhausted false
 *       whose end key CouchDB cannot hold.  Other ranges are decided as with LevelDB, over bytewise key order.  254s then take the
 *       stage's undetermined-writer path.
 *       A value of at most 16384 bytes is scanned by one thread, a longer one by one CTA; both give the same verdict.
 *   fabgpu_state_versions, _indexed and _update refuse, with FABGPU_E_ARG and nothing changed, a version for a public key CouchDB cannot
 *       hold.  A removal of one is accepted: a key a 254 transaction writes becomes unknown, and one CouchDB cannot hold is settled by
 *       removing it. */
enum { FABGPU_STATEDB_LEVELDB = 0, FABGPU_STATEDB_COUCHDB = 1 };
int fabgpu_state_database(fabgpu_ctx* ctx, int kind);
/* The ledger's private-data check (validateAndPreparePvtBatch, core/ledger/kvledger/txmgmt/validation/batch_preparer.go:119-188), an
 * opt-in stage after the flags are final: every collection of the private data the caller holds is hashed and compared with the
 * pvt_rwset_hash of the block's public read/write set, and its rwset is decoded as a KVRWSet, on the device.
 *   The private data is one marshalled rwset.TxPvtReadWriteSet per transaction (ledger.TxPvtData.WriteSet, the rwset bytes unchanged):
 *   entry i is pvt_blob[pvt_off[i] .. pvt_off[i+1]) with SeqInBlock seq[i].  flags are the block's n final flags (those of
 *   TRANSACTIONS_FILTER: fabgpu_validate_mvcc's output, or the caller's once some 254s are settled).
 *   status[3i .. 3i+2] receives entry i's outcome as if its transaction were VALID, with the namespace and collection index (in the
 *   entry's order) where it was decided, -1 where none:
 *     0 OK; 1 mismatch: SHA-256(rwset) differs from retrieveHash(namespace, collection) (types.go:62-78) -- the first such collection
 *     in order, every hash of the entry being checked before any rwset is decoded; 2 skipped: no collection of the public set carries
 *     a pvt_rwset_hash (containsPvtWrites, types.go:49-58); 254: an rwset that does not decode (a level the project's reader refuses, a
 *     string that is not UTF-8), outer levels that do not parse, a transaction whose read/write set the walk never reached (a
 *     non-endorser transaction included), or one whose only public hashes are present but empty while the entry holds a collection.
 *   out = {code, seq, ns, coll}: the block's verdict from the entry with the smallest seq whose outcome is 1 or 254 and whose flag is
 *     VALID or 254 (other flags are ignored, :133-135): 1 with its (seq, ns, coll) when its flag is VALID and it mismatches -- the
 *     reference fails the block's commit -- else 254 with its seq (ns = coll = -1); 0 with seq = ns = coll = -1 when no entry decides.
 *   Call it any number of times after fabgpu_validate_wait(slot) (or a blocking fabgpu_validate_block / _envelopes, slot 0) returned
 *   the block and before the slot's next submit, whether or not fabgpu_validate_mvcc ran.  It runs on the slot's stream under the
 *   slot's lock only, touches no table, and returns with the stream synchronised; the caller's arrays are not referenced afterwards.
 *   FABGPU_E_ARG, with a fabgpu_last_error text and nothing enqueued, for a slot without a finished block, n other than the block's
 *   transaction count, a seq >= n or given twice, NULL arrays with a count > 0, and decreasing offsets.
 *   The private update batch and incrementPvtdataVersionIfNeeded are built by fabgpu_block_pvt_updates, which runs this check itself
 *   with the MVCC stage's flags.  Not restated: the gossip coordinator's filtering, eligibility and missing-data bookkeeping. */
int fabgpu_validate_pvtdata(fabgpu_ctx* ctx, int slot, const uint8_t* flags, size_t n, const uint8_t* pvt_blob, const uint32_t* pvt_off,
                            const uint32_t* seq, size_t n_pvt, int32_t* status, int32_t out[4]);
/* The identities the slot's finished block looked up in the MSP table and did not find (creators and endorsers with a signature
 * job), listed on the device: distinct serialized identities, ordered by first appearance -- transaction, then the creator before its
 * endorsers in endorsement order -- as triples (offset, length, first tx), the offset and length in the bytes the slot's block was
 * submitted in.  At most cap triples go to out; *n_out gets the full count.  These are what the peer runs through its MSP
 * (DeserializeIdentity, Validate, SatisfiesPrincipal) and hands to fabgpu_msp_identities_add.  Any number of calls between the slot's
 * fabgpu_validate_wait and its next submit, on the slot's stream; returns synchronised.  FABGPU_E_ARG, with nothing enqueued, for a
 * slot with no finished block and for NULL outputs. */
int fabgpu_block_unknown_identities(fabgpu_ctx* ctx, int slot, uint32_t* out, size_t cap, size_t* n_out);
/* The block's public and hashed update batch, as applyWriteSet leaves it in publicUpdates and hashUpdates for the transactions the
 * MVCC stage left VALID (validation/types.go:81-111, tx_ops.go:18-232): each key a VALID transaction wrote, at most once, with its final
 * operation in the block at version (block_num, tx).  Records of FABGPU_UPDATE_WORDS uint32 words go to rec, at most rec_cap of them:
 *   [0] tx (the version's tx_num)   [1] op: FABGPU_UPDATE_PUT or FABGPU_UPDATE_DELETE
 *   [2] value source: FABGPU_SRC_NONE (a DELETE), FABGPU_SRC_BLOCK (the KVWrite.value or KVWriteHash.value_hash at [10], [11] -- possibly
 *       an earlier VALID transaction's, which a metadata-only write inherits) or FABGPU_SRC_COMMITTED (the peer reads it with GetState /
 *       GetValueHash: no writer of the block put the key before)
 *   [3] metadata source: FABGPU_SRC_NONE (nil), FABGPU_SRC_BLOCK (statemetadata.Serialize of the deciding metadata write's entries, at
 *       meta[[12] .. [12] + [13])) or FABGPU_SRC_COMMITTED (GetStateMetadata / GetPrivateDataMetadataByHash)
 *   [4], [5] namespace; [6], [7] collection (length 0 for a public key); [8], [9] key (the 32-byte key hash for a hashed key): offsets and
 *       lengths in the bytes the slot's block was submitted in
 *   [10], [11] the value (FABGPU_SRC_BLOCK), [12], [13] the metadata bytes (FABGPU_SRC_BLOCK); 0 otherwise.
 * Records come ordered by tx, then by the wire position of that transaction's first write of the key.  n_out[0] gets the full record
 * count and n_out[1] the metadata bytes; at most meta_cap bytes go to meta.  *complete = 1 when the batch is the block's; 0 with no
 * records (the peer builds the batch itself) when a flag is 254 after the stage, the stage left the block open, two digests shared a
 * tag, the table was broken, a record's metadata entries are not canonical (name = 1 then value = 2, each at most once and non-empty,
 * minimal lengths, nothing else), or a record depends on a key the table marks unknown.  The private update batch is
 * fabgpu_block_pvt_updates'.
 * Call it any number of times after fabgpu_validate_mvcc(slot, block_num) returned, until the next fabgpu_validate_mvcc, the next
 * fabgpu_state_versions* call or the slot's next submit; the first call builds the batch on the slot's stream, later ones copy it.
 * Returns synchronised.  FABGPU_E_ARG, with nothing enqueued, when slot and block_num are not those the stage last ran on, after one of
 * those events, and for NULL outputs. */
#define FABGPU_UPDATE_WORDS 14
#define FABGPU_UPDATE_PUT 1
#define FABGPU_UPDATE_DELETE 2
#define FABGPU_SRC_NONE 0
#define FABGPU_SRC_BLOCK 1
#define FABGPU_SRC_COMMITTED 2
int fabgpu_block_updates(fabgpu_ctx* ctx, int slot, uint64_t block_num, uint32_t* rec, size_t rec_cap, uint8_t* meta, size_t meta_cap,
                         size_t n_out[2], int* complete);
/* The bytes deterministicBytesForPubAndHashUpdates (txmgr/update_batch_bytes.go:29-105) returns for the batch fabgpu_block_updates
 * hands back for the same slot and block: the updateBatchBytes of LockBasedTxMgr.ValidateAndPrepare (lockbased_txmgr.go:220-221).
 * The peer passes out[0 .. *n_out) to kvLedger.addBlockCommitHash (kv_ledger.go:621-632) in place of that function's result, and the
 * block's commit hash is SHA-256(varint(len(flags)) || flags || out[0 .. *n_out) || previous commit hash) as before.  The bytes are
 * proto.Marshal(Updates{kvwrites = 1}) of one KVWrite{namespace = 1 string, collection = 2 string, key = 3, isDelete = 4, value = 5,
 * version_bytes = 6} per record (txmgr/updates.proto; proto3, so empty fields and a false isDelete are left out):
 *   order: namespaces bytewise, namespace "" (the channel config) left out; within a namespace its public keys, then its collections
 *     by name; keys bytewise (a hashed key as its 32 raw bytes);
 *   namespace on the first KVWrite of each namespace only, collection on the first of each collection only (never on a public one);
 *   key the record's key; isDelete for a DELETE; value the PUT's value -- the block's, or for a FABGPU_SRC_COMMITTED record the caller's
 *     (an empty value is left out, with isDelete false); version_bytes EncodeOrderPreservingVarUint64(block_num) followed by that of the
 *     record's tx.  Metadata is not part of the bytes.
 * Committed values: value j is val_blob[val_off[j] .. val_off[j + 1]) and belongs to the j-th record, in fabgpu_block_updates' record
 * order, whose value source is FABGPU_SRC_COMMITTED: what the peer reads to commit it anyway (GetState for a public key, GetValueHash
 * for a hashed one).  n_val must be the number of such records.
 * *n_out gets the full length; at most out_cap bytes go to out.  *complete = 1 when the bytes are the block's (an empty batch, or one
 * of namespace "" only, gives 0 bytes); 0 with *n_out = 0 when the batch is incomplete (fabgpu_block_updates' reasons; n_val is then
 * not checked) or an emitted namespace or collection name is not valid UTF-8 (proto.Marshal fails, and with it the reference's commit):
 * the peer builds the bytes itself.
 * Call window and locks as fabgpu_block_updates: after fabgpu_validate_mvcc(slot, block_num), until the next stage, state version call
 * or submit of the slot; it builds the batch first if no call did, and the batch's order once (later calls reuse both).  Returns
 * synchronised, and the caller's arrays are not referenced afterwards.  FABGPU_E_ARG, with a fabgpu_last_error text and nothing of its
 * own enqueued, for fabgpu_block_updates' refusals, an n_val other than the number of FABGPU_SRC_COMMITTED records, decreasing offsets,
 * NULL outputs, and NULL inputs with n_val > 0. */
int fabgpu_block_update_bytes(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* val_blob, const uint32_t* val_off, size_t n_val,
                              uint8_t* out, size_t out_cap, size_t* n_out, int* complete);
/* The block's private update batch, as validateAndPreparePvtBatch leaves it in PvtUpdates (validation/batch_preparer.go:119-160,
 * 341-410), for the block fabgpu_validate_mvcc(slot, block_num) last ran on.  The private data is passed as fabgpu_validate_pvtdata takes
 * it; the call runs that check itself with the stage's own final flags and fills status and out exactly as fabgpu_validate_pvtdata would
 * with them (a peer that runs the MVCC stage calls this instead).  The batch is defined over those flags only: for each transaction left
 * VALID whose entry the check passed (not skipped), in transaction order,
 *   every KVWrite of its KVRWSets, through namespaces, collections and writes in wire order, is a Put of its value (a Delete when
 *     is_delete) at (block_num, tx); a later write of the same (namespace, collection, key) replaces an earlier one, within one
 *     transaction too;
 *   every KVMetadataWrite's (namespace, collection, key) is collected; for each one whose hashed key (SHA-256 of the key) the hashed
 *     batch of fabgpu_block_updates PUTs at (block_num, h), incrementPvtdataVersionIfNeeded (:360-393) renews the latest private value
 *     -- the batch's, else the committed one -- to version (block_num, h) when its version differs and SHA-256 of it equals that PUT's
 *     value hash.  A hashed DELETE, or no hashed record, never renews.
 * Records of FABGPU_PVT_UPDATE_WORDS uint32 words go to rec, at most rec_cap of them; *n_out gets the full count:
 *   [0] tx (the version's tx_num: the deciding write's, or for a renewal the hashed PUT's)
 *   [1] op: FABGPU_UPDATE_PUT, FABGPU_UPDATE_DELETE or FABGPU_UPDATE_RENEW
 *   [2], [3] namespace; [4], [5] collection; [6], [7] key; [8], [9] the value (PUT; 0 otherwise): offsets and lengths in pvt_blob
 *   [10] RENEW: the index of the hashed PUT record in fabgpu_block_updates' records; UINT32_MAX otherwise.
 * PUT and DELETE records are the batch: each key at most once, ordered by the tx of the write that decides it, then by the position of
 * that transaction's first write of the key among its entry's writes.  A renewal the device decided (the latest value is in the batch)
 * is such a PUT with [0] = the hashed record's tx, in the same place.  RENEW records follow, in the order of their hashed records: a
 * metadata-written key not in the private batch whose hashed key the hashed batch PUTs.  The peer resolves each with one
 * GetPrivateData(ns, coll, key): when a value is present, its version is not (block_num, [0]), and SHA-256(value) equals the hashed
 * record's value hash (its bytes in the block, or GetValueHash for FABGPU_SRC_COMMITTED), it puts that value at (block_num, [0]);
 * otherwise nothing.  So the block's commit batch is fabgpu_block_updates' records, these records and one GetPrivateData per RENEW.
 * *complete = 1 when the batch is the block's; 0 with no records (the peer builds it itself; status and out are still filled) when the
 * public and hashed batch is incomplete (fabgpu_block_updates' reasons), out[0] != 0 (the reference fails the commit), a VALID entry
 * has a KVWrite that is not a delete and has no value field (PutValAndMetadata panics on a nil value; a present but empty value is
 * []byte{} and commits), two key digests shared a tag, a renewal the device decides needs a hashed value hash from the committed state,
 * or a renewal would put a private DELETE's nil value (the hashed value hash is SHA-256 of the empty string: the reference panics).
 * Call window and locks as fabgpu_block_updates: after fabgpu_validate_mvcc(slot, block_num), until the next stage, state version call
 * or submit of the slot; it builds the public and hashed batch first if no call did (a later fabgpu_block_updates only copies it).  The
 * private batch is rebuilt on every call, on the slot's stream; returns synchronised, and the caller's arrays are not referenced
 * afterwards.  FABGPU_E_ARG, with a fabgpu_last_error text and nothing enqueued, for fabgpu_block_updates' refusals, a seq >= the
 * block's transaction count or given twice, decreasing offsets, NULL outputs, and NULL inputs with a count > 0. */
#define FABGPU_PVT_UPDATE_WORDS 11
#define FABGPU_UPDATE_RENEW 3
int fabgpu_block_pvt_updates(fabgpu_ctx* ctx, int slot, uint64_t block_num, const uint8_t* pvt_blob, const uint32_t* pvt_off, const uint32_t* seq,
                             size_t n_pvt, int32_t* status, int32_t out[4], uint32_t* rec, size_t rec_cap, size_t* n_out, int* complete);
/* flags[i] receives the validation code of transaction i; *n_tx_out the number of transactions. */
int fabgpu_validate_block(fabgpu_ctx* ctx, const uint8_t* block, size_t block_len, uint8_t* flags, size_t flags_cap, size_t* n_tx_out);
/* Same for a caller that already holds Block.Data.Data as separate byte strings (the Go validator does): `blob` is their
 * concatenation, env_off the (n_env+1)-entry offset table.  Saves the serial walk over the length-prefixed envelopes. */
int fabgpu_validate_envelopes(fabgpu_ctx* ctx, const uint8_t* blob, const uint32_t* env_off, size_t n_env, uint8_t* flags, size_t flags_cap,
                              size_t* n_tx_out);
/* Both calls in two halves over the FABGPU_SLOTS slots, for a committer that keeps several blocks in flight: _async enqueues
 * the copy and every kernel of the block on the slot's stream and returns; fabgpu_validate_wait blocks until the slot's
 * block is done, runs the duplicate-tx-id pass and writes the flags.  The block bytes must stay valid and unchanged until
 * the wait returns (they are copied by DMA and read again by the duplicate pass).  While the GPU works on block k, the
 * copy of block k+1 proceeds: the PCIe transfer (the largest single phase of a block) is hidden across blocks.
 * fabgpu_validate_block / _envelopes are _async + _wait on slot 0. */
int fabgpu_validate_block_async(fabgpu_ctx* ctx, int slot, const uint8_t* block, size_t block_len);
int fabgpu_validate_envelopes_async(fabgpu_ctx* ctx, int slot, const uint8_t* blob, const uint32_t* env_off, size_t n_env);
int fabgpu_validate_wait(fabgpu_ctx* ctx, int slot, uint8_t* flags, size_t flags_cap, size_t* n_tx_out);
/* Optional pinned staging buffer for the block bytes (the H2D copy of a pageable buffer is several times slower); one per slot. */
int fabgpu_block_buffer(fabgpu_ctx* ctx, size_t bytes, uint8_t** out);                      /* slot 0 */
int fabgpu_block_buffer_slot(fabgpu_ctx* ctx, int slot, size_t bytes, uint8_t** out);
/* Times of the last completed block, microseconds.  [0..4] host wall clock: enqueue, (unused), wait for the device,
 * duplicate-tx-id pass, total from submit to flags.  [5..9] CUDA-event times of the device stages (FABGPU_BLOCK_EVENTS=1):
 * H2D + walk + creator resolve + SHA-256, (unused), endorsement resolve + SHA-256, verify kernel(s), block_decide_kernel. */
int fabgpu_block_timing(const fabgpu_ctx* ctx, double out_us[10]);
/* Device SHA-256 of messages given as up to three byte ranges of `buf` each: jobs = n x {off0,off1,off2,len0,len1,len2}
 * (uint32); digests = n x 32 bytes.  (The hash msp identity.Verify computes first: msp/identities.go:178.) */
int fabgpu_sha256_segments(fabgpu_ctx* ctx, const uint8_t* buf, size_t buf_len, const uint32_t* jobs, size_t n, uint8_t* digests);

/* ---- test / bring-up hooks ------------------------------------------------------------------------------ */
/* Device field primitives on arrays: out[i] = op(a[i], b[i]), 32 big-endian bytes each.  op is a code of the table in
 * fabric-mod_b200/csrc/fieldops.cuh (0 fe_mul ... 16); FABGPU_E_ARG for any other value. */
int fabgpu_test_fieldop(fabgpu_ctx* ctx, int op, const uint8_t* a, const uint8_t* b, size_t n, uint8_t* out);
/* Sampled entries of a device point table: out[i] (64 bytes: X then Y, Montgomery form, little-endian 32-bit limbs) =
 * entry (window[i], digit[i]) = digit * 2^(w * window) * P.  key_slot == -1: the generator's table (w = g_window_bits of
 * fabgpu_build_info, digit in [1, 2^w)); key_slot >= 0: the window table in that raw key slot (w = key_window_bits, digit in
 * [1, 2^w)); key_slot <= -2: a small handle from fabgpu_keys_register_small (w and the window count from fabgpu_small_table_info,
 * digit in [1, 2^(w-1)]), FABGPU_E_ARG when the handle is stale.  Reads a small table only after its build has finished. */
int fabgpu_test_table_entries(fabgpu_ctx* ctx, int key_slot, const uint32_t* window, const uint32_t* digit, size_t n, uint8_t* out);
/* The verdict of fabgpu_state_database's CouchDB value check on each of n values (blob with n + 1 offsets): out[i] holds bits
 * 1 the scanner accepts it, 2 the top-level value is an object, 4 a number overflows float64, 8 a number is undecided, 16 a top-level
 * name is reserved; or 32 (with 2 when the top-level value is an object) when a container deeper than 128 opens before any syntax
 * error, as fabric-mod_b200/csrc/couchval.cuh.  path 0 scans as fabgpu_validate_mvcc does (one thread for a value of at most 16384
 * bytes, one CTA for a longer one); 1 forces the one-thread scan, 2 the CTA scan; FABGPU_E_ARG for any other path. */
int fabgpu_test_couch_values(fabgpu_ctx* ctx, const uint8_t* blob, const uint32_t* off, size_t n, int path, uint32_t* out);
/* Phase times of the last fabgpu_bccsp_verify_batch call, microseconds: [0] key-table lookup/registration,
 * [1] staging copy into pinned memory (host gates + packing on the host-gated path), [2] H2D + kernels + D2H (enqueue to
 * completion), [3] status copy-out.  For metrics export
 * (the reference only has a block-level histogram, gossip/metrics/metrics.go:187-194). */
int fabgpu_last_timing(const fabgpu_ctx* ctx, double out_us[4]);
/* Compile-time table shapes: window bits of the fixed-base table of G and of the per-key tables. */
void fabgpu_build_info(int* g_window_bits, int* key_window_bits);
/* Kernel launches issued by this context so far (bench.py's gpu_launches). */
unsigned long long fabgpu_launch_count(const fabgpu_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* FABGPU_ECDSA_H */
