// TEST HELPER (not product code): compiles fabric-mod_b200/csrc/ecdsa_verify.cuh for the host so the exact
// point / window / verify logic the CUDA kernel runs can be checked against the oracle on the GPU-less build
// box.  Only the innermost limb primitives differ between the two builds (PTX on device, uint64_t here); those
// are checked on the GPU by tests/test_gpu_field.py.
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include <utility>
#include "../../fabric-mod_b200/csrc/ecdsa_verify.cuh"
#include "../../fabric-mod_b200/csrc/ecdsa_batchaffine.cuh"
#include "../../fabric-mod_b200/csrc/fieldops.cuh"

using namespace fabgpu;

static std::vector<aff> g_tab;

extern "C" {

void hostsim_build_gtable()
{
    if (!g_tab.empty()) return;
    g_tab.resize((size_t)FAB_G_WINDOWS * FAB_G_ENTRIES);
    // window j's entries from window j-1's by FAB_WG doublings would be faster; this mirrors the device kernel 1:1
    for (int j = 0; j < FAB_G_WINDOWS; j++)
        for (uint32_t d = 1; d <= (uint32_t)FAB_G_ENTRIES; d++)
            g_tab[(size_t)j * FAB_G_ENTRIES + d - 1] = g_table_entry(j, d);
}

// raw table bytes (little-endian limbs, Montgomery form): entries x 64 bytes
size_t hostsim_gtable(const uint8_t** out)
{
    hostsim_build_gtable();
    *out = (const uint8_t*)g_tab.data();
    return g_tab.size() * sizeof(aff);
}

// inputs: n x 32 big-endian bytes each; out[i] = V_INVALID / V_VALID / V_OFFCURVE
void hostsim_verify_batch(const uint8_t* qx, const uint8_t* qy, const uint8_t* e, const uint8_t* r, const uint8_t* s, int n, uint8_t* out)
{
    hostsim_build_gtable();
    for (int i = 0; i < n; i++) {
        size_t o = 32 * (size_t)i;
        out[i] = (uint8_t)ecdsa_verify_one(u256_from_be(qx + o), u256_from_be(qy + o), u256_from_be(e + o),
                                           u256_from_be(r + o), u256_from_be(s + o), g_tab.data());
    }
}

// Same batch through the per-key-table path: one table per distinct key (built with build_key_window, as the device's
// build_key_tables_kernel does), then ecdsa_verify_one_cached.  Keys that are not curve points are reported V_OFFCURVE.
void hostsim_verify_batch_cached(const uint8_t* qx, const uint8_t* qy, const uint8_t* e, const uint8_t* r, const uint8_t* s, int n, uint8_t* out)
{
    hostsim_build_gtable();
    std::vector<std::pair<std::vector<uint8_t>, std::vector<aff>>> cache;
    std::vector<u256> zs(2 * FAB_Q_ENTRIES);
    for (int i = 0; i < n; i++) {
        size_t o = 32 * (size_t)i;
        std::vector<uint8_t> key(qx + o, qx + o + 32);
        key.insert(key.end(), qy + o, qy + o + 32);
        const std::vector<aff>* tab = nullptr;
        for (auto& c : cache) if (c.first == key) tab = &c.second;
        if (!tab) {
            const u256 x = u256_from_be(qx + o), y = u256_from_be(qy + o);
            aff q; bool ok = u256_lt(x, fe_p()) && u256_lt(y, fe_p());
            if (ok) { q.x = fe_to_mont(x); q.y = fe_to_mont(y); ok = aff_on_curve(q); }
            std::vector<aff> t;
            if (ok) {
                t.resize((size_t)FAB_Q_WINDOWS * FAB_Q_ENTRIES);
                if (FAB_Q_TWO_LEVEL) {      // same two-level build as small_tables_kernel + full_tables_kernel
                    const int half = FAB_WQ / 2, nsmall = (1 << half) - 1;
                    std::vector<aff> lo(nsmall), hi(nsmall);
                    for (int j = 0; j < FAB_Q_WINDOWS; j++) {
                        build_multiples(q, FAB_WQ * j, nsmall, lo.data(), zs.data(), zs.data() + nsmall);
                        build_multiples(q, FAB_WQ * j + half, nsmall, hi.data(), zs.data(), zs.data() + nsmall);
                        for (uint32_t x0 = 1; x0 <= (uint32_t)FAB_Q_ENTRIES; x0 += FAB_TAB_CHUNK) {
                            const int cnt = (int)std::min<uint32_t>(FAB_TAB_CHUNK, (uint32_t)FAB_Q_ENTRIES - x0 + 1);
                            build_window_chunk(lo.data(), hi.data(), half, x0, cnt, t.data() + (size_t)j * FAB_Q_ENTRIES);
                        }
                    }
                } else
                for (int j = 0; j < FAB_Q_WINDOWS; j++) build_key_window(q, j, t.data() + (size_t)j * FAB_Q_ENTRIES, zs.data(), zs.data() + FAB_Q_ENTRIES);
            }
            cache.emplace_back(key, std::move(t));
            tab = &cache.back().second;
        }
        if (tab->empty()) { out[i] = (uint8_t)V_OFFCURVE; continue; }
        out[i] = (uint8_t)ecdsa_verify_one_cached(tab->data(), u256_from_be(e + o), u256_from_be(r + o), u256_from_be(s + o), g_tab.data());
    }
}

// The batch-affine path (ecdsa_batchaffine.cuh) with the CTA exchange replayed on the host: signatures are taken in groups of
// GROUP "threads"; each of GROUP / V "lanes" runs ba_inverse_lane over V strided values, exactly as the inverter warp of
// ecdsa_verify_ba_kernel does.  Keys are given as tables built by the same code as hostsim_verify_batch_cached.
}  // extern "C"

static const std::vector<aff>* ba_key_table(std::vector<std::pair<std::vector<uint8_t>, std::vector<aff>>>& cache, const uint8_t* qx, const uint8_t* qy)
{
    std::vector<uint8_t> key(qx, qx + 32);
    key.insert(key.end(), qy, qy + 32);
    for (auto& c : cache) if (c.first == key) return &c.second;
    const u256 x = u256_from_be(qx), y = u256_from_be(qy);
    aff q; bool ok = u256_lt(x, fe_p()) && u256_lt(y, fe_p());
    if (ok) { q.x = fe_to_mont(x); q.y = fe_to_mont(y); ok = aff_on_curve(q); }
    std::vector<aff> t;
    if (ok) {
        std::vector<u256> zs(2 * FAB_Q_ENTRIES);
        t.resize((size_t)FAB_Q_WINDOWS * FAB_Q_ENTRIES);
        for (int j = 0; j < FAB_Q_WINDOWS; j++) build_key_window(q, j, t.data() + (size_t)j * FAB_Q_ENTRIES, zs.data(), zs.data() + FAB_Q_ENTRIES);
    }
    cache.emplace_back(key, std::move(t));
    return &cache.back().second;
}

static void ba_exchange(bool modn, std::vector<u256>& vals, int V)
{
    // [limb][thread] layout like the kernel's shared-memory buffers
    const int T = (int)vals.size(), lanes = T / V;
    std::vector<uint32_t> exa(8 * T), exb(8 * T);
    for (int t = 0; t < T; t++) for (int l = 0; l < 8; l++) exa[l * T + t] = vals[t].v[l];
    for (int g = 0; g < lanes; g++) ba_inverse_lane(modn, exa.data() + g, exb.data() + g, V, lanes, T);
    for (int t = 0; t < T; t++) for (int l = 0; l < 8; l++) vals[t].v[l] = exa[l * T + t];
}

extern "C" {

void hostsim_verify_batch_ba(const uint8_t* qx, const uint8_t* qy, const uint8_t* e, const uint8_t* r, const uint8_t* s, int n, uint8_t* out)
{
    hostsim_build_gtable();
    const int GROUP = 64, V = 8;
    std::vector<std::pair<std::vector<uint8_t>, std::vector<aff>>> cache;
    cache.reserve(4096);
    for (int base = 0; base < n; base += GROUP) {
        struct Th { bool ok = false; const aff* qt = nullptr; u256 ev, rv, sv; BaScratch sc; uint32_t dig[FAB_BA_NP]; uint32_t exc = 0, m1 = 0; jac acc; };
        std::vector<Th> th(GROUP);
        std::vector<u256> vals(GROUP);
        for (int t = 0; t < GROUP; t++) {
            vals[t] = u256_const(1, 0, 0, 0, 0, 0, 0, 0);
            const int i = base + t;
            if (i >= n) continue;
            const size_t o = 32 * (size_t)i;
            const std::vector<aff>* tab = ba_key_table(cache, qx + o, qy + o);
            if (tab->empty()) { out[i] = (uint8_t)V_OFFCURVE; continue; }
            out[i] = (uint8_t)V_INVALID;
            Th& h = th[t];
            h.qt = tab->data();
            h.ev = u256_from_be(e + o); h.rv = u256_from_be(r + o); h.sv = u256_from_be(s + o);
            h.ok = ba_range_ok(h.rv, h.sv);
            if (h.ok) vals[t] = h.sv;
        }
        ba_exchange(true, vals, V);
        for (int t = 0; t < GROUP; t++) {
            Th& h = th[t];
            u256 c = fe_one();
            if (h.ok) {
                ba_scalars(h.ev, h.rv, vals[t], h.dig, 1);
                c = ba_forward(true, FAB_BA_N1, g_tab.data(), h.qt, h.dig, 1, nullptr, 0u, h.sc.pre, h.exc);
            }
            vals[t] = c;
        }
        ba_exchange(false, vals, V);
        for (int t = 0; t < GROUP; t++) {
            Th& h = th[t];
            u256 c = fe_one();
            h.acc = jac_infinity();
            if (h.ok) {
                h.m1 = ba_backward(true, false, FAB_BA_N1, vals[t], g_tab.data(), h.qt, h.dig, 1, nullptr, 0u, h.sc.pre, h.sc.pts, h.acc);
                c = ba_forward(false, FAB_BA_N2, g_tab.data(), h.qt, h.dig, 1, h.sc.pts, h.m1, h.sc.pre, h.exc);
            }
            vals[t] = c;
        }
        ba_exchange(false, vals, V);
        for (int t = 0; t < GROUP; t++) {
            Th& h = th[t];
            if (!h.ok) continue;
            ba_backward(false, true, FAB_BA_N2, vals[t], g_tab.data(), h.qt, h.dig, 1, h.sc.pts, h.m1, h.sc.pre, nullptr, h.acc);
            out[base + t] = (uint8_t)(h.exc ? ecdsa_verify_one_cached(h.qt, h.ev, h.rv, h.sv, g_tab.data()) : final_check(h.acc, h.rv));
        }
    }
}

// Same batch through the small-table tier: per distinct key small_bases + small_window (exactly what small_bases_kernel and
// small_windows_kernel do), then ecdsa_verify_one_small.  A key that is not a curve point gets the all-zero first entry.
void hostsim_verify_batch_small(const uint8_t* qx, const uint8_t* qy, const uint8_t* e, const uint8_t* r, const uint8_t* s, int n, uint8_t* out)
{
    hostsim_build_gtable();
    std::vector<std::pair<std::vector<uint8_t>, std::vector<aff>>> cache;
    for (int i = 0; i < n; i++) {
        size_t o = 32 * (size_t)i;
        std::vector<uint8_t> key(qx + o, qx + o + 32);
        key.insert(key.end(), qy + o, qy + o + 32);
        const std::vector<aff>* tab = nullptr;
        for (auto& c : cache) if (c.first == key) tab = &c.second;
        if (!tab) {
            std::vector<aff> t((size_t)FAB_S_POINTS), bases(FAB_S_WINDOWS);
            memset(t.data(), 0, t.size() * sizeof(aff));
            if (small_bases(u256_from_be(qx + o), u256_from_be(qy + o), bases.data()))
                for (int j = 0; j < FAB_S_WINDOWS; j++) small_window(bases[j], t.data() + (size_t)j * FAB_S_HALF);
            cache.emplace_back(key, std::move(t));
            tab = &cache.back().second;
        }
        out[i] = (uint8_t)ecdsa_verify_one_small(tab->data(), u256_from_be(e + o), u256_from_be(r + o), u256_from_be(s + o), g_tab.data());
    }
}

// field / scalar unit hooks, the op table of fieldops.cuh (the device's fabgpu_test_fieldop); -1 for an unknown op
int hostsim_fieldop(int op, const uint8_t* a, const uint8_t* b, int n, uint8_t* out)
{
    if (op < 0 || op >= FOP_COUNT) return -1;
    for (int i = 0; i < n; i++)
        u256_to_be(fieldop(op, u256_from_be(a + 32 * (size_t)i), u256_from_be(b + 32 * (size_t)i)), out + 32 * (size_t)i);
    return 0;
}

// k*P for affine plain (x,y) and plain scalar k, via the same table + Booth routine the kernel uses; returns affine plain
// coordinates, or all-zero for infinity.
void hostsim_scalar_mul(const uint8_t* k, const uint8_t* px, const uint8_t* py, uint8_t* ox, uint8_t* oy)
{
    aff q; q.x = fe_to_mont(u256_from_be(px)); q.y = fe_to_mont(u256_from_be(py));
    jac tab[16];
    build_q_table(tab, q);
    jac r = scalar_mul_var(u256_from_be(k), tab);
    if (jac_is_infinity(r)) { memset(ox, 0, 32); memset(oy, 0, 32); return; }
    aff a = jac_to_aff(r);
    u256_to_be(fe_from_mont(a.x), ox); u256_to_be(fe_from_mont(a.y), oy);
}

// k*P through P's small table (signed-window recoding check): affine plain coordinates, all-zero for infinity
void hostsim_small_mul(const uint8_t* k, const uint8_t* px, const uint8_t* py, uint8_t* ox, uint8_t* oy)
{
    std::vector<aff> t((size_t)FAB_S_POINTS), bases(FAB_S_WINDOWS);
    memset(ox, 0, 32); memset(oy, 0, 32);
    if (!small_bases(u256_from_be(px), u256_from_be(py), bases.data())) return;
    for (int j = 0; j < FAB_S_WINDOWS; j++) small_window(bases[j], t.data() + (size_t)j * FAB_S_HALF);
    jac r = add_small_table(jac_infinity(), u256_from_be(k), t.data());
    if (jac_is_infinity(r)) return;
    aff a = jac_to_aff(r);
    u256_to_be(fe_from_mont(a.x), ox); u256_to_be(fe_from_mont(a.y), oy);
}

// k*G via the fixed-base table
void hostsim_base_mul(const uint8_t* k, uint8_t* ox, uint8_t* oy)
{
    hostsim_build_gtable();
    jac r = add_fixed_base(jac_infinity(), u256_from_be(k), g_tab.data());
    if (jac_is_infinity(r)) { memset(ox, 0, 32); memset(oy, 0, 32); return; }
    aff a = jac_to_aff(r);
    u256_to_be(fe_from_mont(a.x), ox); u256_to_be(fe_from_mont(a.y), oy);
}

}  // extern "C"
