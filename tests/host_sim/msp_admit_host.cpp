// TEST HELPER (not product code): identity admission's host logic and the unknown-identity listing, on the host.
//   mm_*: the MSP table's host mirror (fabric-mod_b200/csrc/msptable.hpp) as fabgpu_msp_configure / fabgpu_msp_identities_add drive it.
//   uk_list: a block's walk and identity lookups (blockdev.cuh: walk_tx, resolve_job, msp_find) followed by the listing steps of
//            unknownids.cuh -- the functions the CUDA kernels call -- run one job at a time.
// With -DUK_ASAN_MAIN it is a program that lists every block of a corpus file (see main) for the sanitizer run.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "../../fabric-mod_b200/csrc/msptable.hpp"
#include "../../fabric-mod_b200/csrc/unknownids.cuh"

using namespace fabgpu;
using namespace fabgpu::bdev;

extern "C" {

void* mm_new() { return new msptab::Mirror(); }
void mm_free(void* h) { delete (msptab::Mirror*)h; }
void mm_configure(void* h, const uint8_t* blob, const uint32_t* off, int n) { ((msptab::Mirror*)h)->configure(blob, off, n); }
// null on success (the identities are appended), else the refusal text and the mirror is unchanged
const char* mm_add(void* h, const uint8_t* blob, const uint32_t* off, const uint8_t* mb, const uint32_t* mo, const uint8_t* keys, const uint8_t* valid,
                   const int32_t* group, const uint32_t* bits, int n, int groups_on, int bits_on, int* grew)
{
    auto* m = (msptab::Mirror*)h;
    if (const char* err = m->check_add(blob, off, mb, mo, keys, valid, group, bits, n, groups_on != 0, bits_on != 0)) return err;
    std::vector<uint32_t> dirty;
    *grew = n ? m->add(blob, off, n, dirty) : 0;
    return nullptr;
}
int mm_find(void* h, const uint8_t* p, uint32_t n) { return ((msptab::Mirror*)h)->find(p, n); }
// out: identities, slots, occupied slots
void mm_info(void* h, uint64_t* out)
{
    auto* m = (msptab::Mirror*)h;
    out[0] = (uint64_t)m->n(); out[1] = m->size();
    out[2] = 0;
    for (uint64_t v : m->ht_hash) out[2] += v != 0;
}

// The listing of one block against the table `m` holds: triples into out (cap of them), the count into *n_out.  env_off: n_env + 1.
void uk_list(void* h, const uint8_t* block, const uint32_t* env_off, uint32_t n_env, const char* channel, uint32_t* out, uint32_t cap, uint32_t* n_out)
{
    auto* mm = (msptab::Mirror*)h;
    const uint32_t T = n_env, J = T * (1 + BD_ENDS_HINT);
    std::vector<int32_t> key_slot(mm->n() + 1, 0);
    MspDev msp = mm->view();
    msp.key_slot = key_slot.data();
    std::vector<TxDev> txs(T); std::vector<RawJob> raw(J); std::vector<ShaJobD> sha(J + 2 * T);
    std::vector<uint8_t> r(32 * (size_t)J), s(32 * (size_t)J), gate(J); std::vector<int32_t> ks(J), ident(J, -1);
    for (auto& q : raw) { q.tx = 0xffffffffu; q.k = -1; q.ident.off = q.ident.len = 0; }
    JobArrays ja; ja.sha = sha.data(); ja.r = r.data(); ja.s = s.data(); ja.key_slot = ks.data(); ja.identity = ident.data(); ja.qx = ja.qy = nullptr;
    ja.gate_ok = gate.data(); ja.J_cap = J; ja.T = T;
    uint32_t n_end = 0;
    for (uint32_t t = 0; t < T; t++) {
        Seg env; env.off = env_off[t]; env.len = env_off[t + 1] - env_off[t];
        walk_tx(block, env, t, (const uint8_t*)channel, (uint32_t)strlen(channel), txs[t], raw.data(), ja, [&](uint32_t n) { const uint32_t j = T + n_end; n_end += n; return j; });
    }
    const uint32_t jobs = T + (n_end < J - T ? n_end : J - T);
    for (uint32_t j = 0; j < jobs; j++) resolve_job(block, j, raw.data(), msp, ja, txs.data());
    uint32_t slots = 16; while (slots < 2 * J) slots <<= 1;
    std::vector<uint64_t> hash(J); std::vector<uint32_t> index(slots, UK_EMPTY), rep(J), cnt(T + 1), o(3 * (size_t)J);
    std::vector<unsigned long long> first(J);
    UkArrays a;
    a.raw = raw.data(); a.ident = ident.data(); a.txs = txs.data(); a.T = T; a.E_cap = J - T; a.n_end = &n_end; a.hash = hash.data();
    a.index = index.data(); a.index_mask = slots - 1; a.rep = rep.data(); a.first = first.data(); a.cnt = cnt.data(); a.out = o.data();
    for (uint32_t j = 0; j < uk_jobs(a); j++) uk_hash_job(block, a, j);
    // the kernel's threads race for slots; here a fixed order stands in for one of the interleavings
    for (uint32_t j = uk_jobs(a); j-- > 0;) uk_insert_job(block, a, j);
    for (uint32_t t = 0; t < T; t++) uk_count_tx(a, t);
    uint32_t acc = 0;
    for (uint32_t t = 0; t < T; t++) { const uint32_t v = cnt[t]; cnt[t] = acc; acc += v; }
    cnt[T] = acc;
    for (uint32_t t = 0; t < T; t++) uk_emit_tx(a, t);
    *n_out = acc;
    memcpy(out, o.data(), 12 * (size_t)(acc < cap ? acc : cap));
}

}  // extern "C"

#ifdef UK_ASAN_MAIN
// Corpus: u32 records; per record: u32 n_ids, (u32 len, bytes) per identity, u32 channel length, channel, u32 block length, block,
// u32 n_env, n_env + 1 u32 offsets.  Prints one line per record: the triples.  Inputs are copied into exact-size heap buffers (plus
// the word of slack the device's arrays carry) so that an out-of-range read is reported.
static uint32_t rd32(FILE* f) { uint32_t v = 0; if (fread(&v, 4, 1, f) != 1) exit(3); return v; }
static std::vector<uint8_t> rdb(FILE* f, uint32_t n) { std::vector<uint8_t> b(n + 8, 0); if (n && fread(b.data(), 1, n, f) != n) exit(3); b.resize(n); return b; }
int main(int argc, char** argv)
{
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    const uint32_t R = rd32(f);
    for (uint32_t rec = 0; rec < R; rec++) {
        const uint32_t n = rd32(f);
        std::vector<uint8_t> blob; std::vector<uint32_t> off{0};
        for (uint32_t i = 0; i < n; i++) { auto b = rdb(f, rd32(f)); blob.insert(blob.end(), b.begin(), b.end()); off.push_back((uint32_t)blob.size()); }
        blob.resize(blob.size() + 8);
        auto ch = rdb(f, rd32(f)); std::string channel(ch.begin(), ch.end());
        const uint32_t bl = rd32(f);
        uint8_t* block = new uint8_t[bl + 64];
        memset(block + bl, 0, 64);
        if (bl && fread(block, 1, bl, f) != bl) return 3;
        const uint32_t n_env = rd32(f);
        std::vector<uint32_t> eo(n_env + 1);
        for (auto& x : eo) x = rd32(f);
        void* h = mm_new();
        mm_configure(h, blob.data(), off.data(), (int)n);
        std::vector<uint32_t> out(3 * (size_t)(n_env * (1 + BD_ENDS_HINT) + 1));
        uint32_t cnt = 0;
        uk_list(h, block, eo.data(), n_env, channel.c_str(), out.data(), (uint32_t)out.size() / 3, &cnt);
        for (uint32_t i = 0; i < 3 * cnt; i++) printf(i ? " %u" : "%u", out[i]);
        printf("\n");
        mm_free(h);
        delete[] block;
    }
    return 0;
}
#endif
