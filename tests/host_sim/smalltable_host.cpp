// TEST HELPER (not product code): one key's small table built on the host by the same small_bases + small_window code that
// small_bases_kernel and small_windows_kernel run (fabric-mod_b200/csrc/ecdsa_verify.cuh), for tests/test_tablecheck.py.
#include <cstring>
#include <vector>
#include "../../fabric-mod_b200/csrc/ecdsa_verify.cuh"

using namespace fabgpu;

extern "C" {

// out: FAB_S_POINTS x 64 bytes (little-endian limbs, Montgomery form); only the all-zero first entry for a key that is not a curve point
void host_small_table(const uint8_t* px, const uint8_t* py, uint8_t* out)
{
    std::vector<aff> bases(FAB_S_WINDOWS), t((size_t)FAB_S_POINTS);
    memset(t.data(), 0, t.size() * sizeof(aff));
    if (small_bases(u256_from_be(px), u256_from_be(py), bases.data()))
        for (int j = 0; j < FAB_S_WINDOWS; j++) small_window(bases[j], t.data() + (size_t)j * FAB_S_HALF);
    memcpy(out, t.data(), t.size() * sizeof(aff));
}

int host_small_window_bits() { return FAB_WS; }

}  // extern "C"
