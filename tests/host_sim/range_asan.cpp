// TEST HELPER (not product code): the MVCC stage with an ordered key index (range_host.cpp) as a program, for AddressSanitizer /
// UndefinedBehaviorSanitizer runs over a corpus of read/write sets whose range queries carry wire-level mutations.  Corpus (little-endian u32 lengths): n_keys, then per key (len ns, len coll, len key bytes,
// block, tx as u64); n_blocks, then per block T and per transaction (htype u8, tv u8, len, read/write set bytes).  Each block is
// checked at the table's height (an open block is closed first); prints one "flags <hex>" line per block and a summary.
#include <stdio.h>
#include <stdlib.h>

#include <string>

#include "range_host.cpp"

static std::string g;
static size_t g_pos = 0;
static uint32_t u32()
{
    if (g_pos + 4 > g.size()) { fprintf(stderr, "corpus truncated\n"); exit(2); }
    uint32_t v; memcpy(&v, g.data() + g_pos, 4); g_pos += 4; return v;
}
static std::string bytes(uint32_t n)
{
    if (g_pos + n > g.size()) { fprintf(stderr, "corpus truncated\n"); exit(2); }
    std::string s = g.substr(g_pos, n); g_pos += n; return s;
}

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    char buf[65536]; size_t r;
    while ((r = fread(buf, 1, sizeof buf, f)) > 0) g.append(buf, r);
    fclose(f);
    void* s = rh_new(0x1234);
    const uint32_t n_keys = u32();
    std::string nb, cb, kb; std::vector<uint32_t> no{0}, co{0}, ko{0}; std::vector<uint64_t> ver;
    for (uint32_t i = 0; i < n_keys; i++) {
        nb += bytes(u32()); cb += bytes(u32()); kb += bytes(u32());
        no.push_back((uint32_t)nb.size()); co.push_back((uint32_t)cb.size()); ko.push_back((uint32_t)kb.size());
        const uint32_t lo = u32(), hi = u32(), tlo = u32(), thi = u32();
        ver.push_back((uint64_t)hi << 32 | lo); ver.push_back((uint64_t)thi << 32 | tlo);
    }
    int failed = 0;
    if (const char* err = rh_apply(s, 2, (const uint8_t*)nb.data(), no.data(), (const uint8_t*)cb.data(), co.data(), (const uint8_t*)kb.data(),
                                   ko.data(), ver.data(), n_keys, 1, 0, 0, &failed)) { fprintf(stderr, "install: %s\n", err); return 1; }
    const uint32_t n_blocks = u32();
    unsigned long long recs = 0, counts[256] = {0};
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t T = u32();
        std::vector<uint8_t> ht(T + 1), tv(T + 1), fl(T + 1);
        std::vector<uint32_t> res(2 * T + 2);
        std::vector<std::string> rw(T);
        std::string blob;
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t head = u32();
            ht[t] = (uint8_t)(head & 0xff); tv[t] = (uint8_t)(head >> 8);
            rw[t] = bytes(u32());
            recs += rw[t].size();
        }
        // the block's read/write sets back to back in an allocation of exactly their length
        for (uint32_t t = 0; t < T; t++) blob += rw[t];
        uint8_t* base = (uint8_t*)malloc(blob.size() ? blob.size() : 1);
        memcpy(base, blob.data(), blob.size());
        size_t off = 0;
        for (uint32_t t = 0; t < T; t++) { res[2 * t] = (uint32_t)off; res[2 * t + 1] = (uint32_t)rw[t].size(); off += rw[t].size(); }
        unsigned long long info[4];
        rh_info(s, info);
        const char* err = rh_mvcc(s, base, res.data(), ht.data(), info[2], tv.data(), fl.data(), T, 0, &failed);
        if (err && strstr(err, "open")) {
            rh_apply(s, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, info[2] + 1, 0, 0, &failed);
            rh_info(s, info);
            err = rh_mvcc(s, base, res.data(), ht.data(), info[2], tv.data(), fl.data(), T, 0, &failed);
        }
        if (err) { fprintf(stderr, "block %u: %s\n", b, err); return 1; }
        free(base);
        printf("flags");
        for (uint32_t t = 0; t < T; t++) { printf(" %02x", fl[t]); counts[fl[t]]++; }
        printf(" .\n");
    }
    unsigned long long info[4];
    rh_info(s, info);
    printf("blocks %u bytes %llu valid %llu conflict %llu undecided %llu keys %llu unknown %llu\n", n_blocks, recs, counts[0], counts[11], counts[254],
           info[0], info[3]);
    unsigned long long ix[3];
    rh_index_info(s, ix);
    printf("index %llu %llu\n", ix[0], ix[1]);
    rh_free(s);
    return 0;
}
