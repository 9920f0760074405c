// TEST HELPER (not product code): fabgpu_validate_pvtdata in the tests' host build -- the scan, check and verdict steps of pvtdata.cuh
// run one item at a time in the order the library launches them, with the library's record-count rerun and its composition of the
// block's verdict.  The device hashes with sha256.cuh's kernel; here a plain SHA-256 does.  The transactions come in as TxDev fields
// (results segment, header type).  Built as a library, or with PV_ASAN_MAIN as a program reading a corpus (tests/test_pvt_asan.py).
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../fabric-mod_b200/csrc/pvtdata.cuh"

using namespace fabgpu::bdev;

namespace {

void sha256(const uint8_t* m0, size_t n, uint8_t out[32])
{
    static const uint32_t K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
        0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
        0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
        0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
        0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
        0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    std::vector<uint8_t> m(m0, m0 + n);
    const uint64_t bits = 8 * (uint64_t)n;
    m.push_back(0x80);
    while (m.size() % 64 != 56) m.push_back(0);
    for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(bits >> (8 * i)));
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    auto rotr = [](uint32_t x, int k) { return (x >> k) | (x << (32 - k)); };
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

}  // namespace

extern "C" {

// The stage over one block: results holds 2T (offset, length) pairs into `block`, htype the header types.  status: 3 per entry, out: the
// verdict as fabgpu_validate_pvtdata writes it.  The argument refusals are the library's (tested through it); entries here are valid.
void pv_host(const uint8_t* block, const uint32_t* results, const uint8_t* htype, size_t T, const uint8_t* flags, const uint8_t* pvt,
             const uint32_t* off, const uint32_t* seq, size_t n_pvt, int32_t* status, int32_t* out)
{
    out[0] = PV_OK; out[1] = out[2] = out[3] = -1;
    if (n_pvt == 0) return;
    std::vector<TxDev> txs(T);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    const uint32_t E = (uint32_t)n_pvt;
    std::vector<uint8_t> ent(E);
    std::vector<uint32_t> first(E), nrec(E);
    uint32_t R_cap = 0, ctr[4];
    std::vector<PvRec> rec; std::vector<ShaJobP> jobs; std::vector<uint8_t> dig;
    unsigned long long verdict = ~0ull;
    PvArrays a;
    a.pvt = pvt; a.off = off; a.seq = seq; a.n_pvt = E; a.flags = flags; a.ent = ent.data(); a.first = first.data(); a.n_rec = nrec.data();
    a.ctr = ctr; a.status = status; a.verdict = &verdict;
    for (;;) {
        rec.resize(R_cap + 1); jobs.resize(R_cap + 1); dig.resize(32 * (R_cap + 1));
        a.rec = rec.data(); a.R_cap = R_cap; a.jobs = jobs.data(); a.dig = dig.data();
        ctr[0] = 0;
        for (uint32_t e = 0; e < E; e++) pv_scan_entry(block, txs.data(), e, a);
        if (ctr[0] <= R_cap) break;
        R_cap = ctr[0];
    }
    for (uint32_t i = 0; i < ctr[0]; i++) sha256(pvt + jobs[i].off[0], jobs[i].len[0], dig.data() + 32 * (size_t)i);
    for (uint32_t i = 0; i < ctr[0]; i++) pv_check_rec(block, txs.data(), i, a);
    for (uint32_t e = 0; e < E; e++) pv_verdict_entry(e, a);
    if (verdict != ~0ull) {
        const uint32_t e = (uint32_t)verdict, s = (uint32_t)(verdict >> 32);
        const int32_t* es = status + 3 * (size_t)e;
        const bool mismatch = es[0] == PV_MISMATCH && flags[s] == TXC_VALID;
        out[0] = mismatch ? PV_MISMATCH : PV_UNDET; out[1] = (int32_t)s;
        out[2] = mismatch ? es[1] : -1; out[3] = mismatch ? es[2] : -1;
    }
}

}  // extern "C"

#ifdef PV_ASAN_MAIN
// Corpus: u32 blocks; per block u32 T, per transaction u32 (htype | flag << 8) and a length-prefixed TxReadWriteSet, then u32 n_pvt and
// per entry u32 seq and a length-prefixed TxPvtReadWriteSet.  Prints each block's verdict and its entries' status, one line per block.
// Every buffer is allocated at its exact length, so a read past any message's end is caught.
int main(int argc, char** argv)
{
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<uint8_t> all;
    uint8_t buf[65536]; size_t k;
    while ((k = fread(buf, 1, sizeof buf, f)) > 0) all.insert(all.end(), buf, buf + k);
    fclose(f);
    size_t p = 0;
    auto u32 = [&]() { uint32_t v; memcpy(&v, all.data() + p, 4); p += 4; return v; };
    const uint32_t nb = u32();
    for (uint32_t b = 0; b < nb; b++) {
        const uint32_t T = u32();
        std::vector<uint8_t> blob, htype(T + 1), flags(T + 1);
        std::vector<uint32_t> results(2 * T + 2);
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t hf = u32(), len = u32();
            htype[t] = (uint8_t)hf; flags[t] = (uint8_t)(hf >> 8);
            results[2 * t] = (uint32_t)blob.size(); results[2 * t + 1] = len;
            blob.insert(blob.end(), all.begin() + p, all.begin() + p + len); p += len;
        }
        const uint32_t E = u32();
        std::vector<uint8_t> pb;
        std::vector<uint32_t> off(E + 1, 0), seq(E + 1);
        for (uint32_t e = 0; e < E; e++) {
            seq[e] = u32(); const uint32_t len = u32();
            pb.insert(pb.end(), all.begin() + p, all.begin() + p + len); p += len;
            off[e + 1] = (uint32_t)pb.size();
        }
        uint8_t* blk = new uint8_t[blob.size() ? blob.size() : 1];
        uint8_t* pv = new uint8_t[pb.size() ? pb.size() : 1];
        if (!blob.empty()) memcpy(blk, blob.data(), blob.size());
        if (!pb.empty()) memcpy(pv, pb.data(), pb.size());
        std::vector<int32_t> status(3 * (size_t)E + 3);
        int32_t out[4];
        pv_host(blk, results.data(), htype.data(), T, flags.data(), pv, off.data(), seq.data(), E, status.data(), out);
        printf("%d %d %d %d", out[0], out[1], out[2], out[3]);
        for (uint32_t e = 0; e < E; e++) printf(" %d %d %d", status[3 * e], status[3 * e + 1], status[3 * e + 2]);
        printf("\n");
        delete[] blk; delete[] pv;
    }
    return 0;
}
#endif
