// Kernels of the device-side block pre-pass (logic in blockdev.cuh): one thread per transaction.
#pragma once
#include <cuda_runtime.h>
#include "blockdev.cuh"

namespace fabgpu { namespace bdev {

// Walks every envelope (one thread per transaction): structure checks, SHA-256 job descriptors, raw signature jobs.
// Creator jobs sit at the transaction's own index; endorsement jobs are appended after them through one atomic counter.
__global__ void __launch_bounds__(32)
block_walk_kernel(const uint8_t* __restrict__ block, const uint32_t* __restrict__ env_off, uint32_t t0, uint32_t count, uint32_t T,
                  const uint8_t* __restrict__ channel, uint32_t channel_len, TxDev* __restrict__ txs, RawJob* __restrict__ raw, JobArrays ja,
                  uint32_t* __restrict__ n_end)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;      // transactions [t0, t0 + count) of the T in the block
    if (i >= count) return;
    const uint32_t t = t0 + i;
    Seg env; env.off = env_off[2 * t]; env.len = env_off[2 * t + 1] - env_off[2 * t];      // (begin, end) pairs
    walk_tx(block, env, t, channel, channel_len, txs[t], raw, ja, [&](uint32_t n) { return T + atomicAdd(n_end, n); });
}

// One thread per signature job: identity lookup, DER / low-S gate, verify operands.
__global__ void __launch_bounds__(64)
block_resolve_kernel(const uint8_t* __restrict__ block, const RawJob* __restrict__ raw, uint32_t j0, uint32_t count, MspDev msp, JobArrays ja,
                     TxDev* __restrict__ txs, const uint32_t* __restrict__ count_dev = nullptr)
{
    if (count_dev) count = min(count, *count_dev);                 // endorsement jobs: as many as the walk emitted
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;      // jobs [j0, j0 + count)
    if (i >= count) return;
    resolve_job(block, j0 + i, raw, msp, ja, txs);
}

// Replays the reference's decision order for every transaction on the verification bitmask and the digests.  lscc_seen (v1.3 mode,
// else null): set when an lscc invocation of the block is flagged 254 (lscc_mark).  txids: the committed tx-id set as it stood when the
// block was submitted; slots null and broken 0 = none installed.
__global__ void __launch_bounds__(128)
block_decide_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, uint32_t T, MspDev msp, PolicyDev pol,
                    const uint32_t* __restrict__ mask, const uint8_t* __restrict__ gate_ok, const int32_t* __restrict__ job_identity,
                    const uint8_t* __restrict__ digests, uint32_t J_cap,
                    uint8_t* __restrict__ flags, uint64_t* __restrict__ txid_hash, Seg* __restrict__ txid_seg, KlArrays kl,
                    uint32_t* __restrict__ lscc_seen, TxidSetDev txids)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    uint64_t h = 0;
    if (kl.w) kl_mark(block, t, txs[t], kl);
    const uint8_t f = decide_tx(block, txs[t], t, msp, pol, [&](uint32_t j) { return gate_ok[j] && ((mask[j >> 5] >> (j & 31)) & 1u); }, job_identity, digests,
                                J_cap, &h, kl.w ? &kl : nullptr, txids.slots || txids.broken ? &txids : nullptr);
    flags[t] = f;
    if (lscc_seen) lscc_mark(txs[t], f, lscc_seen);
    txid_hash[t] = h;
    txid_seg[t] = txs[t].txid_ascii;
}

// Key policy table installed: the resolve stage.  One CTA: the marked transactions (a dependency, or metadata writes) are compacted by a
// block-wide scan, then one thread runs kl_resolve_step over them in index order, so a chain sees final flags; each step costs the
// transaction's own records.
__global__ void __launch_bounds__(256)
block_kl_resolve_kernel(const TxDev* __restrict__ txs, uint32_t T, KlArrays kl, uint8_t* __restrict__ flags)
{
    __shared__ uint32_t warp_sum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, per = (T + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(T, tid * per), hi = min(T, lo + per);
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; t++) c += kl.conflicted[t] != 0;
    uint32_t x = c;                                                 // inclusive scan within the warp, then over the warps
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t v = lane < blockDim.x / 32 ? warp_sum[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += y; }
        warp_sum[lane] = v;
    }
    __syncthreads();
    uint32_t off = x - c + (warp ? warp_sum[warp - 1] : 0);
    for (uint32_t t = lo; t < hi; t++) if (kl.conflicted[t]) kl.clist[off++] = t;
    const uint32_t total = warp_sum[31];
    __syncthreads();
    if (tid != 0) return;
    for (uint32_t k = 0; k < total; k++) kl_resolve_step(kl.clist[k], txs, kl, flags);
}

// fabgpu_committed_txids / _add: one thread per id of the call (ids distinct within the call).  *count += the ids that were new.
__global__ void __launch_bounds__(256)
txid_insert_kernel(TxidSlot* __restrict__ tab, uint32_t mask, uint64_t seed, const TxidSlot* __restrict__ rec, uint32_t n,
                   unsigned long long* __restrict__ count)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = rec[i].w[k];
    if (txid_insert(tab, mask, seed, w, rec[i].state) == 1) atomicAdd(count, 1ull);
}

// Growth: one thread per slot of the old table re-inserts its id into the new one
__global__ void __launch_bounds__(256)
txid_rehash_kernel(TxidSlot* __restrict__ tab, uint32_t mask, uint64_t seed, const TxidSlot* __restrict__ old, uint64_t n_old)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_old) return;
    const uint32_t st = old[i].state;
    if (st < TXID_COMMITTED) return;
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = old[i].w[k];
    txid_insert(tab, mask, seed, w, st);
}

// fabgpu_key_policies_update: writes the changed slots of the key policy table
__global__ void __launch_bounds__(256)
kp_scatter_kernel(KpSlot* __restrict__ slots, const uint32_t* __restrict__ idx, const KpSlot* __restrict__ val, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) slots[idx[i]] = val[i];
}

// fabgpu_msp_identities_add: writes the changed slots of the MSP table's identity index (hash and identity of each)
__global__ void __launch_bounds__(256)
msp_scatter_kernel(uint64_t* __restrict__ ht_hash, int32_t* __restrict__ ht_idx, const uint32_t* __restrict__ pos, const uint64_t* __restrict__ hash,
                   const int32_t* __restrict__ idx, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { ht_hash[pos[i]] = hash[i]; ht_idx[pos[i]] = idx[i]; }
}

// ---- bccsp-level batch with the gates on the device (SURVEY.md section 8f rank 3) ------------------------------------------
// One thread per signature: sw.CSP.Verify's argument gates (bccsp/sw/impl.go:249-257), UnmarshalECDSASignature + IsLowS
// (bccsp/utils/ecdsa.go:43-92) and hashToInt, straight from the raw DER / digest blobs.  pre[i] = 0 hands the signature to
// the verify kernel; any other value is already the final FABGPU_ST_* status.
__global__ void __launch_bounds__(128)
bccsp_gate_kernel(const uint8_t* __restrict__ sigs, const uint32_t* __restrict__ sig_off, const uint8_t* __restrict__ digs,
                  const uint32_t* __restrict__ dig_off, const int32_t* __restrict__ key_idx, const int32_t* __restrict__ slot_of,
                  const uint8_t* __restrict__ keys_xy, int32_t K, uint32_t n, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                  uint8_t* __restrict__ e, int32_t* __restrict__ key_slot, uint8_t* __restrict__ qx, uint8_t* __restrict__ qy,
                  uint8_t* __restrict__ pre, uint32_t sig_base, uint32_t dig_base)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t ki = key_idx[i];
    // the offset tables are the caller's (absolute); `sigs` / `digs` hold the bytes from sig_base / dig_base on (a chunk of a call)
    const uint32_t so = sig_off[i] - sig_base, sl = sig_off[i + 1] - sig_off[i], dof = dig_off[i] - dig_base, dl = dig_off[i + 1] - dig_off[i];
    uint8_t rr[32], ss[32];
    int st;
    if (ki < 0) st = 2;                       // nil key
    else if (sl == 0) st = 3;                 // empty signature
    else if (dl == 0) st = 4;                 // empty digest
    else if (ki >= K) st = 9;                 // not a key of the table
    else st = gate_signature_status(sigs + so, sl, rr, ss);
    uint32_t* r4 = reinterpret_cast<uint32_t*>(r + 32 * (size_t)i);
    uint32_t* s4 = reinterpret_cast<uint32_t*>(s + 32 * (size_t)i);
    if (st != 0) {
        for (int k = 0; k < 8; k++) { r4[k] = 0; s4[k] = 0; }
        key_slot[i] = -1;
        pre[i] = (uint8_t)st;
        return;
    }
    // hashToInt for a 256-bit order: leftmost min(len, 32) bytes, left-padded
    uint8_t ee[32];
    const uint32_t take = dl > 32 ? 32 : dl;
    for (uint32_t k = 0; k < 32 - take; k++) ee[k] = 0;
    for (uint32_t k = 0; k < take; k++) ee[32 - take + k] = digs[dof + k];
    uint32_t* e4 = reinterpret_cast<uint32_t*>(e + 32 * (size_t)i);
#pragma unroll
    for (int k = 0; k < 8; k++) {                                 // 32-bit stores instead of 96 byte stores
        r4[k] = (uint32_t)rr[4 * k] | ((uint32_t)rr[4 * k + 1] << 8) | ((uint32_t)rr[4 * k + 2] << 16) | ((uint32_t)rr[4 * k + 3] << 24);
        s4[k] = (uint32_t)ss[4 * k] | ((uint32_t)ss[4 * k + 1] << 8) | ((uint32_t)ss[4 * k + 2] << 16) | ((uint32_t)ss[4 * k + 3] << 24);
        e4[k] = (uint32_t)ee[4 * k] | ((uint32_t)ee[4 * k + 1] << 8) | ((uint32_t)ee[4 * k + 2] << 16) | ((uint32_t)ee[4 * k + 3] << 24);
    }
    const int32_t slot = slot_of[ki];
    key_slot[i] = slot;
    if (slot == -1 && qx) {                                       // only the generic arithmetic reads the key itself
        for (int k = 0; k < 32; k++) { qx[32 * (size_t)i + k] = keys_xy[64 * (size_t)ki + k]; qy[32 * (size_t)i + k] = keys_xy[64 * (size_t)ki + 32 + k]; }
    }
    pre[i] = 0;
}

__global__ void __launch_bounds__(256)
bccsp_status_kernel(const uint8_t* __restrict__ pre, const uint32_t* __restrict__ mask, const uint32_t* __restrict__ off, uint32_t n,
                    uint8_t* __restrict__ status)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t p = pre[i];
    if (p != 0) { status[i] = p; return; }
    const bool ok = (mask[i >> 5] >> (i & 31)) & 1u, oc = (off[i >> 5] >> (i & 31)) & 1u;
    status[i] = ok ? 0 : (oc ? 10 : 1);       // VALID / ERR_OFF_CURVE / INVALID
}

} }  // namespace fabgpu::bdev
