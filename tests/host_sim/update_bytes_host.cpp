// TEST HELPER (not product code): the update bytes (updatebytes.cuh) in the tests' host build -- updates_host.cpp's stage and batch,
// then the steps one item at a time in the order fabgpu_block_update_bytes launches them, a warp's lanes as one lane.  Built as a
// library of its own, or with UPDATE_BYTES_MAIN as a program for AddressSanitizer / UndefinedBehaviorSanitizer runs over a corpus of
// blocks and committed values.
#include "updates_host.cpp"
#include "../../fabric-mod_b200/csrc/updatebytes.cuh"

#include <utility>

extern "C" {

// hs_updates over the block (block_len bytes), then the bytes: at most out_cap go to out, *n_out = the full length, *complete as
// fabgpu_block_update_bytes gives it.  Null or the refusal text.
const char* hs_update_bytes(void* p, const uint8_t* block, size_t block_len, const uint32_t* results, const uint8_t* htype, unsigned long long block_num,
                            const uint8_t* tv, uint8_t* flags, size_t T, const uint8_t* val_blob, const uint32_t* val_off, size_t n_val, uint8_t* out,
                            size_t out_cap, size_t* n_out, int* complete)
{
    *n_out = 0; *complete = 0;
    const size_t rec_cap = block_len + 16;                         // a record takes a write of the block: at least one byte
    std::vector<uint32_t> rec(rec_cap * UD_WORDS);
    size_t nu[2] = {0, 0}; int ucomplete = 0;
    if (const char* err = hs_updates(p, block, results, htype, block_num, tv, flags, T, rec.data(), rec_cap, nullptr, 0, nu, &ucomplete)) return err;
    if (!ucomplete) return nullptr;
    const uint32_t n = (uint32_t)nu[0];
    std::vector<UbItem> item(n + 1), item2(n + 1);
    std::vector<uint32_t> cidx(n + 1), chunk(n + 1);
    std::vector<unsigned long long> off(n + 1);
    uint32_t ctr[2] = {0, 0};
    UbArrays a;
    a.rec = rec.data(); a.n = n; a.blk = block; a.item = item.data(); a.cidx = cidx.data(); a.cval = val_blob; a.coff = val_off; a.block_num = block_num;
    a.off = off.data(); a.chunk = chunk.data(); a.out = nullptr; a.ctr = ctr;
    // the order
    for (uint32_t i = 0; i < n; i++) cidx[i] = ub_item_rec(i, a) ? 1 : 0;
    UbItem* in = item.data(); UbItem* o2 = item2.data();
    for (uint32_t width = 1; width < n; width <<= 1) {
        for (uint32_t i = 0; i < n; i++) ri_sort_one(in, i, n, width, block, o2);
        std::swap(in, o2);
    }
    a.item = in;
    for (uint32_t i = 0, c = 0; i < n; i++) { const uint32_t f = cidx[i]; cidx[i] = c; c += f; ctr[1] = c; }
    if (n_val != ctr[1]) return "n_val is not the number of the batch's records whose value source is FABGPU_SRC_COMMITTED";
    *complete = 1;
    if (n == 0) return nullptr;
    // the bytes
    for (uint32_t q = 0; q < n; q++) ub_size(q, a);
    unsigned long long b = 0; uint32_t c = 0;
    for (uint32_t q = 0; q < n; q++) { const unsigned long long x = off[q]; const uint32_t y = chunk[q]; off[q] = b; chunk[q] = c; b += x; c += y; }
    off[n] = b; chunk[n] = c;
    if (ctr[0]) { *complete = 0; return nullptr; }
    std::vector<uint8_t> bytes(b + 1, 0xAA);
    a.out = bytes.data();
    for (uint32_t q = 0; q < n; q++) ub_emit(q, a, 0, 1);
    for (uint32_t k = 0; k < c; k++) ub_long(k, a, 0, 1);
    *n_out = b;
    if (std::min<size_t>(b, out_cap)) memcpy(out, bytes.data(), std::min<size_t>(b, out_cap));
    return nullptr;
}

}  // extern "C"

#ifdef UPDATE_BYTES_MAIN
// Corpus (little-endian u32): n_blocks, then per block: block_num (2 words, low first), T, per transaction (htype | tv << 8, len, read/
// write set bytes), then n_val, the n_val lengths and the values' bytes; the table starts empty at the first block's height.  Prints one
// line per block: "block <b> complete <c> <hex of the bytes>".
#include <stdio.h>
#include <string>

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::string g; char buf[65536]; size_t r;
    while ((r = fread(buf, 1, sizeof buf, f)) > 0) g.append(buf, r);
    fclose(f);
    size_t pos = 0;
    auto u32 = [&]() { uint32_t v = 0; if (pos + 4 <= g.size()) memcpy(&v, g.data() + pos, 4); pos += 4; return v; };
    void* s = hs_new(7);
    int failed = 0;
    uint32_t z[2] = {0, 0}; uint8_t zb[1] = {0}; uint64_t zv[2] = {0, 0};
    const uint32_t nb = u32();
    for (uint32_t b = 0; b < nb && pos < g.size(); b++) {
        const unsigned long long lo = u32(), hi = u32(), block_num = lo | hi << 32;
        if (b == 0) hs_apply(s, 1, zb, z, zb, z, zb, z, zv, 0, block_num, 64, 0, &failed);
        const uint32_t T = u32();
        std::vector<uint8_t> tv(T + 1), ht(T + 1), flags(T + 1); std::vector<uint32_t> res(2 * T + 2); std::string blob;
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t h = u32(), len = u32();
            ht[t] = (uint8_t)(h & 0xff); tv[t] = (uint8_t)(h >> 8);
            res[2 * t] = (uint32_t)blob.size() + 8; res[2 * t + 1] = len;
            blob += std::string(8, '\0') + g.substr(std::min(pos, g.size()), len); pos += len;
        }
        blob += std::string(64, '\0');
        const uint32_t nv = u32();
        std::vector<uint32_t> voff(nv + 1, 0);
        for (uint32_t j = 0; j < nv; j++) voff[j + 1] = voff[j] + u32();
        std::vector<uint8_t> vals(g.begin() + std::min(pos, g.size()), g.begin() + std::min(pos + voff[nv], g.size()));
        vals.resize(voff[nv] + 1);
        pos += voff[nv];
        std::vector<uint8_t> bb(blob.begin(), blob.end());
        size_t n_out = 0; int complete = 0;
        std::vector<uint8_t> out(1 << 20);
        if (((HS*)s)->open) hs_apply(s, 0, zb, z, zb, z, zb, z, zv, 0, block_num, 0, 0, &failed);
        const char* err = hs_update_bytes(s, bb.data(), bb.size(), res.data(), ht.data(), block_num, tv.data(), flags.data(), T, vals.data(), voff.data(), nv,
                                          out.data(), out.size(), &n_out, &complete);
        if (err) { printf("block %u refused %s\n", b, err); continue; }
        printf("block %u complete %d ", b, complete);
        for (size_t i = 0; i < std::min(n_out, out.size()); i++) printf("%02x", out[i]);
        printf("\n");
    }
    hs_free(s);
    return 0;
}
#endif
