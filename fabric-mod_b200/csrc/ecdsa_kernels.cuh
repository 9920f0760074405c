// CUDA kernels for the batch verifier (sm_90a).  See ecdsa_verify.cuh for the per-signature algorithm.
#pragma once
#include <cuda_runtime.h>
#include "ecdsa_verify.cuh"
#include "ecdsa_batchaffine.cuh"
#include "fieldops.cuh"

namespace fabgpu {

// Launch shapes (tools/kbench.py times them at 64k and 256k batches): both kernels are pipe-bound, not
// latency-bound, so occupancy variants differ by a few per cent.
#ifndef FAB_VERIFY_THREADS
#define FAB_VERIFY_THREADS 448        // largest CTA of the generic kernel (launch_verify picks 64 / 256 / 448 by batch size)
#endif
#ifndef FAB_VERIFY_MINBLOCKS
#define FAB_VERIFY_MINBLOCKS 1
#endif

// 32 big-endian bytes at a 16-byte aligned address -> limbs, as two 128-bit loads + byte permutes
__device__ __forceinline__ u256 load_be32(const uint8_t* p)
{
    const uint4 hi = __ldg(reinterpret_cast<const uint4*>(p));        // bytes 0..15  (most significant)
    const uint4 lo = __ldg(reinterpret_cast<const uint4*>(p) + 1);    // bytes 16..31
    u256 r;
    r.v[7] = __byte_perm(hi.x, 0, 0x0123); r.v[6] = __byte_perm(hi.y, 0, 0x0123);
    r.v[5] = __byte_perm(hi.z, 0, 0x0123); r.v[4] = __byte_perm(hi.w, 0, 0x0123);
    r.v[3] = __byte_perm(lo.x, 0, 0x0123); r.v[2] = __byte_perm(lo.y, 0, 0x0123);
    r.v[1] = __byte_perm(lo.z, 0, 0x0123); r.v[0] = __byte_perm(lo.w, 0, 0x0123);
    return r;
}

// Builds the fixed-base table: one thread per (window, digit).
__global__ void build_g_table_kernel(aff* gtab)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int total = FAB_G_WINDOWS * FAB_G_ENTRIES;
    if (idx >= total) return;
    const int j = idx / FAB_G_ENTRIES;
    const uint32_t d = (uint32_t)(idx % FAB_G_ENTRIES) + 1u;
    gtab[idx] = g_table_entry(j, d);
}

// One signature per thread.  SoA inputs: n x 32 big-endian bytes each.  Output: bit i%32 of word i/32 is 1 iff
// signature i is VALID; offcurve (optional) flags public keys that are not curve points.
// key_slot (optional): signatures whose key has a precomputed table (slot >= 0) were decided by
// ecdsa_verify_cached_kernel; this kernel skips them and ORs its bits into the words that kernel wrote.
__global__ void __launch_bounds__(FAB_VERIFY_THREADS, FAB_VERIFY_MINBLOCKS)
ecdsa_verify_kernel(const int32_t* __restrict__ key_slot, const uint8_t* __restrict__ qx, const uint8_t* __restrict__ qy,
                    const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s, uint32_t n,
                    const aff* __restrict__ gtab, uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve,
                    const uint32_t* __restrict__ n_dev, uint32_t n_base)
{
    if (n_dev) n = min(n, n_base + *n_dev);      // batch size decided by an earlier kernel of the stream (block path): n is the launch bound
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t res = V_INVALID;
    if (idx < n && (key_slot == nullptr || key_slot[idx] < 0)) {
        const size_t o = (size_t)idx * 32;
        res = ecdsa_verify_one(load_be32(qx + o), load_be32(qy + o), load_be32(e + o), load_be32(r + o), load_be32(s + o), gtab);
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, res == V_VALID);
    const uint32_t omask = __ballot_sync(0xffffffffu, res == V_OFFCURVE);
    if ((threadIdx.x & 31u) == 0 && idx < n) {
        if (key_slot) { mask[idx >> 5] |= vmask; if (offcurve) offcurve[idx >> 5] |= omask; }
        else { mask[idx >> 5] = vmask; if (offcurve) offcurve[idx >> 5] = omask; }
    }
}

// ---- mixed batches: signatures without a big key table, compacted by class ------------------------------------------------------
// key_slot codes (device side, after the host resolved the handles): >= 0 slot of a big window table (ecdsa_verify_cached_kernel);
// -1 no table (generic arithmetic: 255 doublings); <= -2 small table number -2 - code (ecdsa_verify_small_kernel).
// In a batch where only SOME keys own a big table the generic kernel used to run over all n threads and return at once for the tabled
// ones; with the kinds interleaved every warp still walked the whole generic path for its untabled lanes: a half-and-half batch cost as
// much as an all-generic one.  Now the indices are compacted first (warp-aggregated append): the untabled
// ones from the front of idx[0, n), the small-table ones from its back; counters at idx[n] and idx[n + 1].  Each class then runs over
// whole warps; results are OR-ed into the mask words the big-table kernel wrote (bit 0 for everything that is not its own).
__global__ void compact_classes_kernel(const int32_t* __restrict__ key_slot, uint32_t n, uint32_t* __restrict__ idx, uint32_t* __restrict__ counts,
                                       const uint32_t* __restrict__ n_dev, uint32_t n_base)
{
    const uint32_t cap = n;                                    // the small-table indices grow down from idx[cap - 1]
    if (n_dev) n = min(n, n_base + *n_dev);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t ks = i < n ? key_slot[i] : 0;
    const bool g = ks == -1, sm = ks <= -2;
    const uint32_t mg = __ballot_sync(0xffffffffu, g), ms = __ballot_sync(0xffffffffu, sm);
    if ((mg | ms) == 0) return;
    const uint32_t lane = threadIdx.x & 31u, below = (1u << lane) - 1u;
    uint32_t bg = 0, bs = 0;
    if (lane == 0) { if (mg) bg = atomicAdd(counts, (uint32_t)__popc(mg)); if (ms) bs = atomicAdd(counts + 1, (uint32_t)__popc(ms)); }
    bg = __shfl_sync(0xffffffffu, bg, 0); bs = __shfl_sync(0xffffffffu, bs, 0);
    if (g) idx[bg + __popc(mg & below)] = i;
    if (sm) idx[cap - 1u - (bs + __popc(ms & below))] = i;
}

#ifndef FAB_INDEXED_THREADS
#define FAB_INDEXED_THREADS 128
#endif
__global__ void __launch_bounds__(FAB_INDEXED_THREADS, 3)
ecdsa_verify_indexed_kernel(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ count, const uint8_t* __restrict__ qx, const uint8_t* __restrict__ qy,
                            const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s, const aff* __restrict__ gtab,
                            uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= *count) return;
    const uint32_t i = idx[t];
    const size_t o = (size_t)i * 32;
    const uint32_t res = ecdsa_verify_one(load_be32(qx + o), load_be32(qy + o), load_be32(e + o), load_be32(r + o), load_be32(s + o), gtab);
    if (res == V_VALID) atomicOr(mask + (i >> 5), 1u << (i & 31u));
    else if (res == V_OFFCURVE && offcurve) atomicOr(offcurve + (i >> 5), 1u << (i & 31u));
}

// ---- small key tables (ecdsa_verify.cuh: FAB_WS, ecdsa_verify_one_small) ---------------------------------------------------------
#ifndef FAB_SMALL_THREADS
#define FAB_SMALL_THREADS 512         // largest CTA the kernel may be launched with (launch_small picks the shape by batch size, like launch_verify)
#endif
#ifndef FAB_SMALL_MINBLOCKS
#define FAB_SMALL_MINBLOCKS 1
#endif
// idx != NULL: thread t takes signature idx[cap - 1 - t] for t < *count (the small-table list of compact_classes_kernel) and ORs its
// verdict into the mask; idx == NULL: every signature of [0, n) has a small table (key_slot[i] <= -2), one ballot word per warp.
__global__ void __launch_bounds__(FAB_SMALL_THREADS, FAB_SMALL_MINBLOCKS)
ecdsa_verify_small_kernel(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ count, uint32_t cap, const int32_t* __restrict__ key_slot,
                          const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s, uint32_t n,
                          const aff* __restrict__ gtab, const aff* __restrict__ stab, uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const bool act = idx ? (t < *count) : (t < n);
    const uint32_t i = (idx && act) ? idx[cap - 1u - t] : t;
    uint32_t res = V_INVALID;
    if (act) {                                                     // one call site: a single expanded copy of the verification
        const size_t o = (size_t)i * 32;
        res = ecdsa_verify_one_small(stab + (size_t)(-2 - key_slot[i]) * FAB_S_POINTS, load_be32(e + o), load_be32(r + o), load_be32(s + o), gtab);
    }
    if (idx) {
        if (res == V_VALID) atomicOr(mask + (i >> 5), 1u << (i & 31u));
        else if (res == V_OFFCURVE && offcurve) atomicOr(offcurve + (i >> 5), 1u << (i & 31u));
        return;
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, res == V_VALID), omask = __ballot_sync(0xffffffffu, res == V_OFFCURVE);
    if ((threadIdx.x & 31u) == 0 && t < n) { mask[t >> 5] = vmask; if (offcurve) offcurve[t >> 5] = omask; }
}

// Build, stage 1: thread f derives the window bases of key keys_xy[f] (small_bases) into bases[f][.]; a key that is not a curve
// point gets an all-zero bases[f][0] AND an all-zero first table entry (what ecdsa_verify_one_small reports as off-curve).
__global__ void small_bases_kernel(const uint8_t* __restrict__ keys_xy, const int32_t* __restrict__ slots, int nkeys, aff* __restrict__ bases,
                                   aff* __restrict__ stab)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nkeys) return;
    aff* b = bases + (size_t)f * FAB_S_WINDOWS;
    if (!small_bases(load_be32(keys_xy + 64 * (size_t)f), load_be32(keys_xy + 64 * (size_t)f + 32), b)) {
        aff z; z.x = u256_zero(); z.y = u256_zero();
        b[0] = z;
        stab[(size_t)slots[f] * FAB_S_POINTS] = z;
    }
}
// Stage 2: thread (f, j) fills window j of the key's table (small_window).
__global__ void __launch_bounds__(128)
small_windows_kernel(const aff* __restrict__ bases, const int32_t* __restrict__ slots, int nkeys, aff* __restrict__ stab)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nkeys * FAB_S_WINDOWS) return;
    const int f = t / FAB_S_WINDOWS, j = t % FAB_S_WINDOWS;
    const aff first = bases[(size_t)f * FAB_S_WINDOWS];
    if (u256_is_zero(first.x) && u256_is_zero(first.y)) return;
    small_window(bases[t], stab + (size_t)slots[f] * FAB_S_POINTS + (size_t)j * FAB_S_HALF);
}

// ---- validity-bitmask exchange over peer memory (one process per GPU; SURVEY.md section 8e) -----------------------------------
// Every rank owns a receive buffer (cudaMalloc'ed, exported through CUDA IPC, mapped by all peers): `gens` generations of
// world x words_per_rank mask words, then world step flags.  The verify kernel's epilogue stores each warp's ballot word into
// the buffer of EVERY rank (plain st.global on peer-mapped addresses: P2P writes over NVLink / NVSwitch); the last CTA to finish
// publishes the step number into every rank's flag array; peer_wait_kernel (same stream) then spins until the flags of all ranks
// have reached the step, i.e. until the whole bitmask has landed locally.  No NCCL call on the data path.
#define FAB_PEER_MAX 8
struct PeerOut {
    uint32_t* buf[FAB_PEER_MAX];   // every rank's receive buffer as mapped in THIS process (buf[rank] is the local one)
    uint32_t* done;                // local counter of finished CTAs (device memory, zero between launches)
    uint32_t world, rank;
    uint32_t words_per_rank;       // mask words each rank contributes
    uint32_t gen_off;              // word offset of this step's generation inside a buffer
    uint32_t flag_off;             // word offset of the flag array inside a buffer
    uint32_t step;                 // published when this rank's words are all written
};

__device__ __forceinline__ void peer_store_word(const PeerOut& po, uint32_t word_index, uint32_t v)
{
    const uint32_t at = po.gen_off + po.rank * po.words_per_rank + word_index;
#pragma unroll
    for (uint32_t p = 0; p < FAB_PEER_MAX; p++) if (p < po.world) po.buf[p][at] = v;      // static indices: the parameter stays in constant memory
}

// Called by every thread of a CTA after its mask words are stored: the last CTA of the grid publishes the step.  ONE system-scope
// fence per CTA, by thread 0 after the barrier (fences are cumulative: the barrier orders the warp leaders' peer stores before it).  The
// first version fenced in every thread -- 64k system fences per launch, each waiting for its peer writes to be acknowledged.
__device__ __forceinline__ void peer_publish(const PeerOut& po)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const uint32_t prev = atomicAdd(po.done, 1u);
        if (prev == gridDim.x - 1) {
            *po.done = 0u;                                // ready for the next launch (stream order)
            __threadfence_system();
#pragma unroll
            for (uint32_t p = 0; p < FAB_PEER_MAX; p++) if (p < po.world) *reinterpret_cast<volatile uint32_t*>(po.buf[p] + po.flag_off + po.rank) = po.step;
        }
    }
}

// Waits (on the stream) until every rank has published `step`; gives up after ~2 s and records that in *timeout_flag so a
// dead peer can never hang the GPU (the host reads the flag and reports a device error: the caller falls back).
__global__ void peer_wait_kernel(const uint32_t* flags, uint32_t world, uint32_t step, uint32_t* timeout_flag)
{
    const uint32_t p = threadIdx.x;
    if (p >= world) return;
    const long long t0 = clock64();
    while ((int32_t)(*reinterpret_cast<const volatile uint32_t*>(flags + p) - step) < 0) {
        if (clock64() - t0 > 4000000000ll) { *timeout_flag = 1u; break; }
        __nanosleep(40);
    }
}

// Fallback for launches whose mask was produced by several kernels (mixed key-table / generic batches): copy the finished local
// words to every peer, then publish.
__global__ void peer_scatter_kernel(const uint32_t* __restrict__ local_words, uint32_t n_words, PeerOut po)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_words) peer_store_word(po, i, local_words[i]);
    peer_publish(po);
}

// ---- scalars of the key-table kernel, one shared inversion per CTA ---------------------------------------------------------------
// ecdsa_prep_kernel runs before ecdsa_verify_cached_kernel on the same stream, one thread per signature: the range gate r, s in
// [1, n-1], w = s^-1 by Montgomery's trick over the CTA (ba_inverse_lane, mod n: one warp of division-step inversions serves
// FAB_PREP_THREADS signatures), then u1 = e w and u2 = r w.  A signature that fails the gate contributes 1 to the product and gets
// u2 = 0, which no signature that passes it can have (r, w in [1, n-1] and n is prime): the chain kernel reads that as INVALID.
// Signatures without a window table (key_slot < 0: mixed batches) contribute 1 too and get nothing written; the chain kernel skips them.
// Scalars: 64 bytes per signature as four rows of uint4 -- [u1 limbs 0..3], [u1 4..7], [u2 0..3], [u2 4..7] -- each row `stride`
// entries long (the launch bound n), so that every load and store of a warp is one contiguous 512-byte span.
// The kernel needs few registers: several CTAs stay resident per SM, and while one CTA's warps wait for its inverter warp the others'
// products and loads run.  (The `ba` kernels shared their inversions inside the 128-register chain kernel: one CTA per SM, seven of
// eight warps idle at each exchange.)
#ifndef FAB_PREP_THREADS
#define FAB_PREP_THREADS 128           // signatures per shared inversion (DESIGN.md section 4.1: 64 / 128 / 256 measured)
#endif
#ifndef FAB_PREP_MINBLOCKS
#define FAB_PREP_MINBLOCKS 6           // 128 threads x 80 registers (no spills): six CTAs per SM
#endif
__global__ void __launch_bounds__(FAB_PREP_THREADS, FAB_PREP_MINBLOCKS)
ecdsa_prep_kernel(const int32_t* __restrict__ key_slot, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                  uint32_t n, uint4* __restrict__ scal, const uint32_t* __restrict__ n_dev, uint32_t n_base)
{
    constexpr int T = FAB_PREP_THREADS;
    __shared__ uint32_t exa[8 * T], exb[8 * T];                // [limb][thread], as ba_cta_inverse
    const uint32_t stride = n;
    if (n_dev) n = min(n, n_base + *n_dev);
    if (blockIdx.x * T >= n) return;                            // whole CTA past the device-side batch size (block path)
    const int tid = threadIdx.x;
    const uint32_t idx = blockIdx.x * T + tid;
    const size_t o = (size_t)idx * 32;
    const bool mine = idx < n && key_slot[idx] >= 0;           // signatures without a window table are not the chain kernel's
    bool ok = false;
    u256 rv = u256_zero(), v = u256_const(1, 0, 0, 0, 0, 0, 0, 0);
    if (mine) {
        rv = load_be32(r + o);
        const u256 sv = load_be32(s + o);
        ok = ba_range_ok(rv, sv);
        if (ok) v = sv;
    }
#pragma unroll
    for (int l = 0; l < 8; l++) exa[l * T + tid] = v.v[l];
    __syncthreads();
    if (tid < 32) ba_inverse_lane(true, exa + tid, exb + tid, T / 32, 32, T);     // inverter lane l: values l, l + 32, l + 64, ...
    __syncthreads();
    if (!mine) return;
    u256 u1 = u256_zero(), u2 = u256_zero();
    if (ok) {
        u256 w;
#pragma unroll
        for (int l = 0; l < 8; l++) w.v[l] = exa[l * T + tid];
        ecdsa_u1u2(load_be32(e + o), rv, w, u1, u2);
    }
    scal[idx] = make_uint4(u1.v[0], u1.v[1], u1.v[2], u1.v[3]);
    scal[stride + idx] = make_uint4(u1.v[4], u1.v[5], u1.v[6], u1.v[7]);
    scal[2 * (size_t)stride + idx] = make_uint4(u2.v[0], u2.v[1], u2.v[2], u2.v[3]);
    scal[3 * (size_t)stride + idx] = make_uint4(u2.v[4], u2.v[5], u2.v[6], u2.v[7]);
}

// The scalars ecdsa_prep_kernel wrote for signature idx, read where the chain uses them: u2 is not held in registers through u1's windows.
struct ScalRows {
    const uint4* scal;
    uint32_t stride, idx;
    __device__ u256 operator()(int t) const
    {
        const uint4 a = __ldg(scal + (size_t)(2 * t) * stride + idx), b = __ldg(scal + (size_t)(2 * t + 1) * stride + idx);
        return u256_const(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
    }
};

#ifndef FAB_CACHED_THREADS
#define FAB_CACHED_THREADS 512        // largest CTA the kernel may be launched with (launch_verify picks 128 / 256 / 512)
#endif
#ifndef FAB_CACHED_MINBLOCKS
#define FAB_CACHED_MINBLOCKS 1        // 512 threads x 128 registers = one CTA per SM; four CTAs of 128 threads fit as well
#endif
// Signatures whose public key has a precomputed window table: both scalar multiplications are fixed-base
// (FAB_G_WINDOWS + FAB_Q_WINDOWS mixed additions gathered from HBM-resident tables, no doublings), on the scalars ecdsa_prep_kernel
// wrote (same n, n_dev, n_base).  Slot < 0 -> bit 0, left to ecdsa_verify_kernel.  qtab: key_slot_capacity tables of
// FAB_Q_WINDOWS*FAB_Q_ENTRIES affine points.
__global__ void __launch_bounds__(FAB_CACHED_THREADS, FAB_CACHED_MINBLOCKS)
ecdsa_verify_cached_kernel(const int32_t* __restrict__ key_slot, const uint4* __restrict__ scal, const uint8_t* __restrict__ r,
                           uint32_t n, const aff* __restrict__ gtab, const aff* __restrict__ qtab,
                           uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve, const uint32_t* __restrict__ n_dev, uint32_t n_base, PeerOut po)
{
    const uint32_t stride = n;
    if (n_dev) n = min(n, n_base + *n_dev);
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t res = V_INVALID;
    if (idx < n) {
        const int32_t slot = key_slot[idx];
        if (slot >= 0) {
            const ScalRows sc = {scal, stride, idx};
            if (!u256_is_zero(sc(1))) {                             // u2 = 0: r or s outside [1, n-1]
                const xyzz acc = ecdsa_chain_cached(qtab + (size_t)slot * (FAB_Q_WINDOWS * FAB_Q_ENTRIES), sc, gtab);
                res = final_check(acc, load_be32(r + (size_t)idx * 32));     // r loaded after the chain: no registers held through it
            }
        }
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, res == V_VALID);
    if ((threadIdx.x & 31u) == 0 && idx < n) {
        mask[idx >> 5] = vmask;
        if (offcurve) offcurve[idx >> 5] = 0u;
        if (po.world) peer_store_word(po, idx >> 5, vmask);      // fused epilogue: the ballot word goes to every rank's buffer (P2P stores)
    }
    if (po.world) peer_publish(po);
}

// ---- lane-split variant of the Jacobian-chain kernel (the "warp-cooperative" shape of BASELINE.json's north_star, measured) ----
// LANES adjacent lanes share one signature BY WINDOWS: lane l accumulates windows l, l + LANES, l + 2 LANES, ... of the 12 + 16
// table windows into its own Jacobian partial sum (no carry ever crosses a lane), the partial sums are tree-combined with the
// complete addition through shuffles, lane 0 of the group runs the final check.  w = s^-1 and u1, u2 are computed by every lane
// of the group (in SIMT that costs the same as computing them in one lane and broadcasting).  Thread count x LANES, chain length
// per thread / LANES.  It measured slower than one signature per thread and stays selectable for comparison.
#ifndef FAB_LANES_THREADS
#define FAB_LANES_THREADS 256
#endif
template <int LANES>
__global__ void __launch_bounds__(FAB_LANES_THREADS, 2)
ecdsa_verify_lanes_kernel(const int32_t* __restrict__ key_slot, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                          const uint8_t* __restrict__ s, uint32_t n, const aff* __restrict__ gtab, const aff* __restrict__ qtab,
                          uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve)
{
    constexpr int T = FAB_LANES_THREADS, SIGS = T / LANES, NW = FAB_G_WINDOWS + FAB_Q_WINDOWS, STEPS = (NW + LANES - 1) / LANES;
    __shared__ uint32_t dig[(STEPS * LANES) * SIGS];           // [window][signature of the CTA]: table entry index or FAB_BA_INF
    const int lane = threadIdx.x % LANES, sg = threadIdx.x / LANES;
    const uint32_t idx = blockIdx.x * SIGS + sg;
    bool ok = false;
    const aff* qt = qtab;
    u256 rv;
    if (idx < n) {
        const int32_t slot = key_slot[idx];
        if (slot >= 0) {
            const size_t o = (size_t)idx * 32;
            qt = qtab + (size_t)slot * (FAB_Q_WINDOWS * FAB_Q_ENTRIES);
            rv = load_be32(r + o);
            const u256 sv = load_be32(s + o);
            ok = ba_range_ok(rv, sv);
            if (ok) {
                const u256 w = sc_inv_to_mont_safegcd(sv);
                const u256 u1 = sc_mul(sc_reduce_once(load_be32(e + o)), w), u2 = sc_mul(rv, w);
                if (lane == 0) {                                   // one lane publishes the digits of all windows
                    uint32_t kk[8];
#pragma unroll
                    for (int i = 0; i < 8; i++) kk[i] = u1.v[i];
#pragma unroll
                    for (int j = 0; j < FAB_G_WINDOWS; j++) {
                        const uint32_t d = kk[0] & (uint32_t)FAB_G_ENTRIES;
#pragma unroll
                        for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WG) | (kk[i + 1] << (32 - FAB_WG));
                        kk[7] >>= FAB_WG;
                        dig[j * SIGS + sg] = d ? (uint32_t)j * (uint32_t)FAB_G_ENTRIES + (d - 1u) : FAB_BA_INF;
                    }
#pragma unroll
                    for (int i = 0; i < 8; i++) kk[i] = u2.v[i];
#pragma unroll
                    for (int j = 0; j < FAB_Q_WINDOWS; j++) {
                        const uint32_t d = kk[0] & (uint32_t)FAB_Q_ENTRIES;
#pragma unroll
                        for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WQ) | (kk[i + 1] << (32 - FAB_WQ));
                        kk[7] >>= FAB_WQ;
                        dig[(FAB_G_WINDOWS + j) * SIGS + sg] = d ? (uint32_t)j * (uint32_t)FAB_Q_ENTRIES + (d - 1u) : FAB_BA_INF;
                    }
                    for (int j = NW; j < STEPS * LANES; j++) dig[j * SIGS + sg] = FAB_BA_INF;
                }
            }
        }
    }
    __syncwarp();                                                  // a group never straddles a warp (LANES divides 32)
    jac acc = jac_infinity();
    if (ok) {
#pragma unroll 1
        for (int t = 0; t < STEPS; t++) {
            const int j = t * LANES + lane;
            const uint32_t di = dig[j * SIGS + sg];
            if (di != FAB_BA_INF) acc = jac_add_aff_t<FAB_CACHED_INLINE != 0>(acc, load_aff_nc((j < FAB_G_WINDOWS ? gtab : qt) + di));
        }
    }
    // tree-combine the partial sums of the group's lanes
#pragma unroll
    for (int d = 1; d < LANES; d <<= 1) {
        jac o;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            o.X.v[i] = __shfl_xor_sync(0xffffffffu, acc.X.v[i], d);
            o.Y.v[i] = __shfl_xor_sync(0xffffffffu, acc.Y.v[i], d);
            o.Z.v[i] = __shfl_xor_sync(0xffffffffu, acc.Z.v[i], d);
        }
        if (ok && (lane & (2 * d - 1)) == 0) acc = jac_add(acc, o);
    }
    const uint32_t res = (ok && lane == 0) ? final_check(acc, rv) : V_INVALID;
    const uint32_t b = __ballot_sync(0xffffffffu, res == V_VALID);
    // bits of lanes 0, LANES, 2 LANES, ... -> 32 / LANES consecutive mask bits
    uint32_t packed = 0;
#pragma unroll
    for (int k = 0; k < 32 / LANES; k++) packed |= ((b >> (k * LANES)) & 1u) << k;
    if ((threadIdx.x & 31u) == 0) {
        const uint32_t first = blockIdx.x * SIGS + (threadIdx.x / LANES);     // first signature of this warp
        // Every warp whose slice lies in a mask word of the batch writes it, also when all its signatures are past n: a warp covers
        // only 32 / LANES signatures, and the rest of the batch's last word would otherwise keep whatever the buffer held.
        if ((first >> 5) <= ((n - 1) >> 5)) {
            if (LANES == 2) { reinterpret_cast<uint16_t*>(mask)[first >> 4] = (uint16_t)packed; if (offcurve) reinterpret_cast<uint16_t*>(offcurve)[first >> 4] = 0; }
            else if (LANES == 4) { reinterpret_cast<uint8_t*>(mask)[first >> 3] = (uint8_t)packed; if (offcurve) reinterpret_cast<uint8_t*>(offcurve)[first >> 3] = 0; }
            else { mask[first >> 5] = packed; if (offcurve) offcurve[first >> 5] = 0; }
        }
    }
}

// ---- batch-affine key-table kernel (ecdsa_batchaffine.cuh) ----
#ifndef FAB_BA_THREADS
#define FAB_BA_THREADS 256            // signatures (= threads) per CTA; the shared inversion is amortised over this many
#endif
#ifndef FAB_BA_MINBLOCKS
#define FAB_BA_MINBLOCKS 2
#endif
#ifndef FAB_BA_INVWARPS
#define FAB_BA_INVWARPS 1             // warps that run the shared inversion of a round (each lane: THREADS / (32 INVWARPS) values)
#endif
#ifndef FAB_BA_SMS
#define FAB_BA_SMS 132
#endif
#ifndef FAB_BA_STAGGER_NS
#define FAB_BA_STAGGER_NS 0           // CTAs that share an SM start this many ns apart (x their index modulo the residency): while one
#endif                                // CTA waits for its inverter warp, the other is in a compute phase instead of waiting in step

// The shared inversion of one exchange round, run by the lanes of the round's inverter warp(s): out of line, ONE copy for the
// three rounds and both moduli.
__device__ __noinline__ void ba_inverter(bool modn, uint32_t* val, uint32_t* tmp)
{
    ba_inverse_lane(modn, val, tmp, FAB_BA_THREADS / (32 * FAB_BA_INVWARPS), 32 * FAB_BA_INVWARPS, FAB_BA_THREADS);
}

// One exchange round: every thread contributes v, the round's inverter warps invert all FAB_BA_THREADS values with Montgomery's
// trick (ba_inverse_lane), every thread gets its own inverse back.  exa / exb: 8 x FAB_BA_THREADS words each, [limb][thread].
__device__ __forceinline__ u256 ba_cta_inverse(bool modn, const u256& v, uint32_t* exa, uint32_t* exb, int round)
{
    constexpr int T = FAB_BA_THREADS, W = T / 32, K = FAB_BA_INVWARPS;
    const int tid = threadIdx.x;
#pragma unroll
    for (int l = 0; l < 8; l++) exa[l * T + tid] = v.v[l];
    __syncthreads();
    const int first = (round * K + (int)blockIdx.x) % W;
    const int rank = ((tid >> 5) - first + W) % W;             // this warp's position among the round's inverter warps
    if (rank < K) {
        const int g = rank * 32 + (tid & 31);                  // handles values g, g + 32 K, g + 64 K, ...
        ba_inverter(modn, exa + g, exb + g);
    }
    __syncthreads();
    u256 r;
#pragma unroll
    for (int l = 0; l < 8; l++) r.v[l] = exa[l * T + tid];
    return r;
}

// The complete per-signature routine for the (never expected) zero-denominator case; out of line, shares nothing with the hot path.
__device__ __noinline__ uint32_t ba_fallback_verify(const aff* qtab, const uint8_t* e, const uint8_t* r, const uint8_t* s, const aff* gtab)
{
    return ecdsa_verify_one_cached(qtab, load_be32(e), load_be32(r), load_be32(s), gtab);
}

// Same contract as ecdsa_verify_cached_kernel (one signature per thread, SoA inputs, ballot mask out); the CTA must be
// FAB_BA_THREADS wide.  Three exchange rounds: s^-1 mod n, the denominators of level 1, the denominators of level 2.
__global__ void __launch_bounds__(FAB_BA_THREADS, FAB_BA_MINBLOCKS)
ecdsa_verify_ba_kernel(const int32_t* __restrict__ key_slot, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                       const uint8_t* __restrict__ s, uint32_t n, const aff* __restrict__ gtab, const aff* __restrict__ qtab,
                       uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve, const uint32_t* __restrict__ n_dev, uint32_t n_base, PeerOut po)
{
    constexpr int T = FAB_BA_THREADS;
    __shared__ uint32_t dig[FAB_BA_NP * T];
    __shared__ uint32_t exa[8 * T], exb[8 * T];
    if (n_dev) n = min(n, n_base + *n_dev);
#if FAB_BA_STAGGER_NS > 0
    {   // CTAs are handed to SMs round-robin: blockIdx / (number of SMs) is this CTA's position among its SM's residents
        const unsigned pos = (blockIdx.x / FAB_BA_SMS) % FAB_BA_MINBLOCKS;
        if (pos) __nanosleep(pos * FAB_BA_STAGGER_NS);
    }
#endif
    const uint32_t idx = blockIdx.x * T + threadIdx.x;
    const size_t o = (size_t)idx * 32;
    const aff* qt = qtab;
    bool ok = false;
    u256 v = u256_const(1, 0, 0, 0, 0, 0, 0, 0);
    if (idx < n) {
        const int32_t slot = key_slot[idx];
        if (slot >= 0) {
            qt = qtab + (size_t)slot * (FAB_Q_WINDOWS * FAB_Q_ENTRIES);
            const u256 sv = load_be32(s + o);
            ok = ba_range_ok(load_be32(r + o), sv);
            if (ok) v = sv;
        }
    }
    uint32_t* mydig = dig + threadIdx.x;
    v = ba_cta_inverse(true, v, exa, exb, 0);                 // w = s^-1 R mod n
    BaScratch sc;
    uint32_t exc = 0, m1 = 0;
    jac acc = jac_infinity();
    if (ok) { ba_scalars(load_be32(e + o), load_be32(r + o), v, mydig, T); ba_prefetch_leaves(mydig, T, gtab, qt); }
#pragma unroll 1
    for (int level = 0; level < 2; level++) {
        const bool first = level == 0;
        const int cnt = first ? FAB_BA_N1 : FAB_BA_N2;
        u256 c = fe_one();
        if (ok) c = ba_forward(first, cnt, gtab, qt, mydig, T, sc.pts, m1, sc.pre, exc);
        c = ba_cta_inverse(false, c, exa, exb, 1 + level);
        if (ok) {
            const uint32_t m = ba_backward(first, !first, cnt, c, gtab, qt, mydig, T, sc.pts, m1, sc.pre, sc.pts, acc);
            if (first) m1 = m;
        }
    }
    uint32_t res = V_INVALID;
    if (ok) res = exc ? ba_fallback_verify(qt, e + o, r + o, s + o, gtab) : final_check(acc, load_be32(r + o));
    const uint32_t vmask = __ballot_sync(0xffffffffu, res == V_VALID);
    if ((threadIdx.x & 31u) == 0 && idx < n) {
        mask[idx >> 5] = vmask;
        if (offcurve) offcurve[idx >> 5] = 0u;
        if (po.world) peer_store_word(po, idx >> 5, vmask);      // fused epilogue: the ballot word goes to every rank's buffer
    }
    if (po.world) peer_publish(po);
}

// ---- batch-affine, two signatures per thread, no CTA exchange (large batches) ------------------------------------------------
// The CTA-shared inversion of ecdsa_verify_ba_kernel costs three barrier rounds during which seven of eight warps wait for the
// inverter warp.  Here a thread carries TWO signatures -- CTA-local
// indices t and t + T -- and runs Montgomery's trick over its own pair: half an inversion per signature and round, no shared
// state, no barrier; warps drift freely, so the scheduler always has independent work.  Half as many threads per batch: the
// launch code uses this kernel only when the batch still fills the machine (see launch_verify).
#ifndef FAB_BA2_THREADS
#define FAB_BA2_THREADS 128
#endif
#ifndef FAB_BA2_MINBLOCKS
#define FAB_BA2_MINBLOCKS 4
#endif
__device__ __noinline__ void ba2_inverse_pair(bool modn, u256& a, u256& b) { ba_inverse_pair(modn, a, b); }
// Out-of-line passes: the kernel body unrolls its two signatures (so that their state stays in registers) without holding two
// copies of the loops.
__device__ __noinline__ u256 ba2_forward(bool first, const aff* gtab, const aff* qt, const uint32_t* dig, BaScratch* sc, uint32_t m1, uint32_t* exc)
{
    uint32_t x = *exc;
    const u256 c = ba_forward(first, first ? FAB_BA_N1 : FAB_BA_N2, gtab, qt, dig, FAB_BA2_THREADS, sc->pts, m1, sc->pre, x);
    *exc = x;
    return c;
}
// level 1: returns the infinity flags of its results; level 2: returns the verdict of the signature
__device__ __noinline__ uint32_t ba2_backward(bool first, const u256& inv, const aff* gtab, const aff* qt, const uint32_t* dig, BaScratch* sc, uint32_t m1,
                                              const uint8_t* r32)
{
    jac acc = jac_infinity();
    const uint32_t m = ba_backward(first, !first, first ? FAB_BA_N1 : FAB_BA_N2, inv, gtab, qt, dig, FAB_BA2_THREADS, sc->pts, m1, sc->pre, sc->pts, acc);
    if (first) return m;
    return final_check(acc, load_be32(r32));
}

__global__ void __launch_bounds__(FAB_BA2_THREADS, FAB_BA2_MINBLOCKS)
ecdsa_verify_ba2_kernel(const int32_t* __restrict__ key_slot, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                        const uint8_t* __restrict__ s, uint32_t n, const aff* __restrict__ gtab, const aff* __restrict__ qtab,
                        uint32_t* __restrict__ mask, uint32_t* __restrict__ offcurve)
{
    constexpr int T = FAB_BA2_THREADS;
    __shared__ uint32_t dig[2 * FAB_BA_NP * T];
    const uint32_t base = blockIdx.x * (2 * T) + threadIdx.x;       // signatures base and base + T
    bool ok[2] = {false, false};
    const aff* qt[2] = {qtab, qtab};
    u256 v[2];
    v[0] = v[1] = u256_const(1, 0, 0, 0, 0, 0, 0, 0);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t idx = base + h * T;
        if (idx < n) {
            const int32_t slot = key_slot[idx];
            if (slot >= 0) {
                qt[h] = qtab + (size_t)slot * (FAB_Q_WINDOWS * FAB_Q_ENTRIES);
                const u256 sv = load_be32(s + (size_t)idx * 32);
                ok[h] = ba_range_ok(load_be32(r + (size_t)idx * 32), sv);
                if (ok[h]) v[h] = sv;
            }
        }
    }
    ba2_inverse_pair(true, v[0], v[1]);                              // w = s^-1 R mod n for both
    BaScratch sc[2];
    uint32_t exc[2] = {0, 0}, m1[2] = {0, 0};
    uint32_t res[2] = {V_INVALID, V_INVALID};
#pragma unroll
    for (int h = 0; h < 2; h++)
        if (ok[h]) {
            ba_scalars(load_be32(e + (size_t)(base + h * T) * 32), load_be32(r + (size_t)(base + h * T) * 32), v[h], dig + h * FAB_BA_NP * T + threadIdx.x, T);
            ba_prefetch_leaves(dig + h * FAB_BA_NP * T + threadIdx.x, T, gtab, qt[h]);
        }
#pragma unroll 1
    for (int level = 0; level < 2; level++) {
        const bool first = level == 0;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            v[h] = fe_one();
            if (ok[h]) v[h] = ba2_forward(first, gtab, qt[h], dig + h * FAB_BA_NP * T + threadIdx.x, &sc[h], m1[h], &exc[h]);
        }
        ba2_inverse_pair(false, v[0], v[1]);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!ok[h]) continue;
            const size_t o = (size_t)(base + h * T) * 32;
            const uint32_t m = ba2_backward(first, v[h], gtab, qt[h], dig + h * FAB_BA_NP * T + threadIdx.x, &sc[h], m1[h], r + o);
            if (first) m1[h] = m;
            else res[h] = exc[h] ? ba_fallback_verify(qt[h], e + o, r + o, s + o, gtab) : m;
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t idx = base + h * T;
        const uint32_t vmask = __ballot_sync(0xffffffffu, res[h] == V_VALID);
        if ((threadIdx.x & 31u) == 0 && idx < n) {
            mask[idx >> 5] = vmask;
            if (offcurve) offcurve[idx >> 5] = 0u;
        }
    }
}

// Key-table build: thread t builds window (t % FAB_Q_WINDOWS) of key (t / FAB_Q_WINDOWS) into the key's slot.
// flags[k] = 1 when key k is a curve point (its table is valid), 0 otherwise (nothing is written for it).
__global__ void build_key_tables_kernel(const uint8_t* __restrict__ keys_xy, const int32_t* __restrict__ slots, int nkeys,
                                        aff* __restrict__ qtab, u256* __restrict__ scratch, uint32_t* __restrict__ flags)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nkeys * FAB_Q_WINDOWS) return;
    const int k = t / FAB_Q_WINDOWS, j = t % FAB_Q_WINDOWS;
    const u256 x = load_be32(keys_xy + 64 * (size_t)k), y = load_be32(keys_xy + 64 * (size_t)k + 32);
    const u256 p = fe_p();
    bool ok = u256_lt(x, p) && u256_lt(y, p);
    aff q;
    if (ok) { q.x = fe_to_mont(x); q.y = fe_to_mont(y); ok = aff_on_curve(q); }
    if (j == 0) flags[k] = ok ? 1u : 0u;
    if (!ok) return;
    u256* zs = scratch + (size_t)t * 2 * FAB_Q_ENTRIES;
    build_key_window(q, j, qtab + ((size_t)slots[k] * FAB_Q_WINDOWS + j) * FAB_Q_ENTRIES, zs, zs + FAB_Q_ENTRIES);
}

// Two-level table build (build_window_chunk in ecdsa_verify.cuh), shared by the per-key tables and the generator's table.
// Stage 1: thread ((k * windows + j) * 2 + h) builds the 2^(wbits/2) - 1 multiples of 2^(wbits j + h wbits/2) P_k into
//   small[thread][.]; scratch: 2 * (2^(wbits/2) - 1) field elements per thread.  keys_xy == NULL: one "key", P = G.
//   flags[k] = 1 when key k is a curve point, 0 otherwise (nothing is built for it).
__global__ void small_tables_kernel(const uint8_t* __restrict__ keys_xy, int nkeys, int wbits, int windows, aff* __restrict__ small,
                                    u256* __restrict__ scratch, uint32_t* __restrict__ flags)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nkeys * windows * 2) return;
    const int k = t / (windows * 2), j = (t / 2) % windows, h = t & 1;
    const int half = wbits / 2, nsmall = (1 << half) - 1;
    aff q;
    if (keys_xy) {
        const u256 x = load_be32(keys_xy + 64 * (size_t)k), y = load_be32(keys_xy + 64 * (size_t)k + 32);
        const u256 p = fe_p();
        bool ok = u256_lt(x, p) && u256_lt(y, p);
        if (ok) { q.x = fe_to_mont(x); q.y = fe_to_mont(y); ok = aff_on_curve(q); }
        if (j == 0 && h == 0) flags[k] = ok ? 1u : 0u;
        if (!ok) return;
    } else { q.x = fe_gx_mont(); q.y = fe_gy_mont(); }
    u256* zs = scratch + (size_t)t * 2 * nsmall;
    build_multiples(q, wbits * j + h * half, nsmall, small + (size_t)t * nsmall, zs, zs + nsmall);
}

// Stage 2: thread ((k * windows + j) * chunks + c) writes FAB_TAB_CHUNK consecutive entries of table slots[k] (slot 0 when
// slots == NULL): one mixed addition each plus one shared inversion.  Runs after stage 1 on the same stream.
__global__ void __launch_bounds__(128)
full_tables_kernel(const aff* __restrict__ small, const int32_t* __restrict__ slots, const uint32_t* __restrict__ flags, int nkeys, int wbits,
                   int windows, aff* __restrict__ tab)
{
    const uint32_t entries = (1u << wbits) - 1u, chunks = (entries + FAB_TAB_CHUNK - 1) / FAB_TAB_CHUNK;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)nkeys * windows * chunks) return;
    const uint32_t c = (uint32_t)(t % chunks);
    const int j = (int)((t / chunks) % windows), k = (int)(t / ((size_t)chunks * windows));
    if (flags && !flags[k]) return;
    const int half = wbits / 2, nsmall = (1 << half) - 1;
    const aff* lo = small + ((size_t)(k * windows + j) * 2) * nsmall;
    const uint32_t x0 = 1u + c * FAB_TAB_CHUNK;
    const int count = (int)min((uint32_t)FAB_TAB_CHUNK, entries - x0 + 1u);
    const size_t slot = slots ? (size_t)slots[k] : 0;
    build_window_chunk(lo, lo + nsmall, half, x0, count, tab + (slot * windows + j) * (size_t)entries);
}

// Test hook: out[i] = entry (window[i], digit[i]) of a table of `stride` entries per window (digit >= 1).
__global__ void table_entries_kernel(const aff* __restrict__ tab, uint32_t stride, const uint32_t* __restrict__ window, const uint32_t* __restrict__ digit,
                                     uint32_t n, aff* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = tab[(size_t)window[i] * stride + (digit[i] - 1u)];
}

// Unit-test hook: out[i] = op(a[i], b[i]) on the device primitives, op from the table of fieldops.cuh (tests/test_gpu_field.py).
__global__ void fieldop_kernel(int op, const uint8_t* a, const uint8_t* b, int n, uint8_t* out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u256 x = load_be32(a + 32 * (size_t)i), y = load_be32(b + 32 * (size_t)i);
    u256_to_be(fieldop(op, x, y), out + 32 * (size_t)i);
}

}  // namespace fabgpu
