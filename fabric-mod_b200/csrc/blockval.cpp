// See blockval.hpp.
#include "blockval.hpp"
#include "blockdev.cuh"

namespace fabgpu { namespace blockval {

// The envelopes are read with the device walk's wire reader (bdev::Reader), so that every level of the block path takes the
// same decision on every tag.
bool split_block(const uint8_t* block, size_t len, std::vector<Seg>& envs)
{
    envs.clear();
    if (len >= (1ull << 32)) return false;                               // offsets are 32-bit
    auto reader = [&](uint32_t off, uint32_t n) { bdev::Reader r; r.base = block; r.pos = off; r.end = off + n; r.ok = true; return r; };
    bdev::Seg data; data.off = data.len = 0; bool has_data = false;
    {
        bdev::Reader r = reader(0, (uint32_t)len);
        uint32_t f, wt; uint64_t v; bdev::Seg b;
        while (r.next(f, wt, v, b)) {
            if (f == 1 || f == 3) { if (wt != 2) return false; }         // header, metadata: known fields, must be length-delimited
            if (f == 2) { if (wt != 2) return false; data = b; has_data = true; }
        }
        if (!r.ok) return false;
    }
    if (!has_data) return true;
    bdev::Reader r = reader(data.off, data.len);
    uint32_t f, wt; uint64_t v; bdev::Seg b;
    while (r.next(f, wt, v, b)) {
        if (f != 1) continue;
        if (wt != 2) return false;
        Seg e; e.off = b.off; e.len = b.len;
        envs.push_back(e);
    }
    return r.ok;
}

} }  // namespace fabgpu::blockval
