// TEST HELPER (not product code): CouchDB's value and key checks (couchval.cuh) as a program, for AddressSanitizer /
// UndefinedBehaviorSanitizer runs.  Corpus (little-endian u32 lengths): n, then per value its length and bytes.  Each value is copied
// into a heap buffer of exactly its length, so a read past its end is caught; prints one line per value: the verdict bits of the
// one-thread scan and of the CTA scan (run lane by lane), and whether cv_key_ok holds for the same bytes.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "../../fabric-mod_b200/csrc/couchval.cuh"

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::string g;
    char buf[65536]; size_t r;
    while ((r = fread(buf, 1, sizeof buf, f)) > 0) g.append(buf, r);
    fclose(f);
    size_t pos = 0;
    auto u32 = [&]() { uint32_t v; if (pos + 4 > g.size()) exit(2); memcpy(&v, g.data() + pos, 4); pos += 4; return v; };
    const uint32_t n = u32();
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t len = u32();
        if (pos + len > g.size()) return 2;
        uint8_t* p = (uint8_t*)malloc(len ? len : 1);
        memcpy(p, g.data() + pos, len);
        pos += len;
        printf("%u %u %d\n", fabgpu::bdev::cv_short(p, len), fabgpu::bdev::cv_long_host(p, len), (int)fabgpu::bdev::cv_key_ok(p, len));
        free(p);
    }
    return 0;
}
