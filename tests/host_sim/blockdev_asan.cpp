// TEST DRIVER (not product code): the block pre-pass's byte-level code -- split_block (blockval.cpp), walk_tx, resolve_job and
// decide_tx (blockdev.cuh) -- over a corpus of blocks read from a file, built with -fsanitize=address,undefined by
// tests/test_blockval_host.py.  Every block's bytes sit in an allocation of exactly their size, so a read past an envelope or the
// block is reported.  Every signature that passes the DER gate counts as verified, so that decide_tx reaches the policy evaluation.
//
// Corpus file (little-endian uint32 lengths and counts):
//   n_ids, then per identity: serialized (len, bytes), MSP id (len, bytes), valid (1 byte)
//   n_nodes, then n_nodes x 4 int32 policy nodes;  n_principals, then per principal (len, bytes);  channel (len, bytes)
//   n_blocks, then per block: ends_hint, serialized common.Block (len, bytes)
// Prints "blocks <n> parsed <n> transactions <n>" and exits 0; any sanitizer report aborts with a non-zero status.
#include <cstdio>
#include <cstdlib>
#include "blockdev_host.cpp"

namespace {

struct In {
    FILE* f;
    uint32_t u32() { uint32_t v; if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "corpus truncated\n"); exit(2); } return v; }
    std::string bytes() { std::string s(u32(), '\0'); if (!s.empty() && fread(&s[0], 1, s.size(), f) != s.size()) { fprintf(stderr, "corpus truncated\n"); exit(2); } return s; }
};

// SHA-256 (FIPS 180-4), for the tx-id and proposal-hash digests decide_tx compares
void sha256(const std::string& m, uint8_t out[32])
{
    static const uint32_t K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3,
        0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
        0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13,
        0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
        0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
        0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    std::string p = m;
    p.push_back((char)0x80);
    while (p.size() % 64 != 56) p.push_back('\0');
    const uint64_t bits = 8ull * m.size();
    for (int i = 7; i >= 0; i--) p.push_back((char)(bits >> (8 * i)));
    auto rotr = [](uint32_t x, int n) { return (x >> n) | (x << (32 - n)); };
    for (size_t blk = 0; blk < p.size(); blk += 64) {
        uint32_t w[64];
        for (int i = 0; i < 16; i++)
            w[i] = (uint32_t)(uint8_t)p[blk + 4 * i] << 24 | (uint32_t)(uint8_t)p[blk + 4 * i + 1] << 16 | (uint32_t)(uint8_t)p[blk + 4 * i + 2] << 8 | (uint8_t)p[blk + 4 * i + 3];
        for (int i = 16; i < 64; i++)
            w[i] = w[i - 16] + (rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3)) + w[i - 7] + (rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10));
        uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
        for (int i = 0; i < 64; i++) {
            const uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i];
            const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(h[i / 4] >> (24 - 8 * (i % 4)));
}

}  // namespace

int main(int argc, char** argv)
{
    if (argc != 2) { fprintf(stderr, "usage: %s corpus\n", argv[0]); return 2; }
    In in{fopen(argv[1], "rb")};
    if (!in.f) { perror(argv[1]); return 2; }
    const uint32_t n_ids = in.u32();
    std::vector<std::string> ser(n_ids), msp(n_ids); std::vector<uint8_t> valid(n_ids);
    for (uint32_t i = 0; i < n_ids; i++) { ser[i] = in.bytes(); msp[i] = in.bytes(); uint8_t v; if (fread(&v, 1, 1, in.f) != 1) return 2; valid[i] = v; }
    const uint32_t n_nodes = in.u32();
    std::vector<int32_t> nodes(4 * n_nodes);
    for (auto& x : nodes) x = (int32_t)in.u32();
    const uint32_t n_pr = in.u32();
    std::vector<std::string> pr(n_pr);
    for (auto& s : pr) s = in.bytes();
    const std::string channel = in.bytes();
    auto blob = [](const std::vector<std::string>& v, std::string& b, std::vector<uint32_t>& off) {
        off.assign(1, 0); for (const auto& s : v) { b += s; off.push_back((uint32_t)b.size()); }
    };
    std::string idb, mb, pb; std::vector<uint32_t> ido, mo, po;
    blob(ser, idb, ido); blob(msp, mb, mo); blob(pr, pb, po);

    const uint32_t n_blocks = in.u32();
    uint32_t parsed = 0; uint64_t n_tx = 0;
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t ends_hint = in.u32();
        const std::string s = in.bytes();
        std::vector<uint8_t> block(s.begin(), s.end());                  // exactly the block's size
        std::vector<fabgpu::blockval::Seg> envs;
        if (!fabgpu::blockval::split_block(block.data(), block.size(), envs)) continue;
        parsed++;
        std::vector<uint8_t> env_blob; std::vector<uint32_t> env_off(1, 0);
        for (const auto& e : envs) { env_blob.insert(env_blob.end(), block.begin() + e.off, block.begin() + e.off + e.len); env_off.push_back((uint32_t)env_blob.size()); }
        env_blob.shrink_to_fit();
        void* h = bd_new((const uint8_t*)idb.data(), ido.data(), (const uint8_t*)mb.data(), mo.data(), valid.data(), (int)n_ids, nodes.data(), (int)n_nodes,
                         (const uint8_t*)pb.data(), po.data(), (int)n_pr, channel.c_str());
        const int T = (int)envs.size();
        const int n_end = bd_plan_ex(h, env_blob.data(), env_off.data(), T, (int)ends_hint, 0);
        std::vector<uint8_t> sig_ok(T + n_end + 1, 0), chk(64 * (size_t)T + 1, 0), flags(T + 1, 0);
        for (int j = 0; j < T + n_end; j++) {
            int ident, gok; uint8_t r[32], sv[32]; uint32_t segs[6];
            bd_job(h, j, &ident, &gok, r, sv, segs);
            sig_ok[j] = ident >= 0 && gok;
        }
        const H* hh = (const H*)h;
        for (int t = 0; t < T; t++) {
            uint32_t segs[12];
            bd_check(h, t, segs);
            for (int q = 0; q < 2; q++) {
                std::string m;
                for (int k = 0; k < 3; k++) m.append((const char*)hh->block.data() + segs[6 * q + k], segs[6 * q + 3 + k]);
                sha256(m, &chk[64 * (size_t)t + 32 * q]);
            }
        }
        bd_decide(h, sig_ok.data(), chk.data(), flags.data());
        bd_free(h);
        n_tx += T;
    }
    fclose(in.f);
    printf("blocks %u parsed %u transactions %llu\n", n_blocks, parsed, (unsigned long long)n_tx);
    return 0;
}
