// TEST DRIVER (not product code): blockdev_keylevel_asan.cpp's sanitizer run in v1.3 mode, so that the v1.3 byte code -- dispatch_plan's
// system-chaincode checks, decide_v13 with the namespace versions, and the block's lscc pass -- runs over the corpus too.  Built with
// -fsanitize=address,undefined by tests/test_v13_asan.py.  Every signature that passes the DER gate counts as verified.
//
// Corpus file: blockdev_keylevel_asan.cpp's, with the namespace table after the key table: n_ns, then per entry name (len, bytes), root
// (int32) and lscc version (len, bytes).  Prints one line per parsed block, "flags <hex> <lscc seen>", then "blocks <n> parsed <n>
// transactions <n> lscc <n>".
#define main blockdev_asan_main
#include "blockdev_asan.cpp"
#undef main
#include "blockdev_keylevel.inc"
#include "blockdev_v13.inc"

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
    const uint32_t n_kn = in.u32();
    std::vector<int32_t> kn(4 * n_kn + 4);
    for (uint32_t i = 0; i < 4 * n_kn; i++) kn[i] = (int32_t)in.u32();
    const uint32_t n_keys = in.u32();
    std::vector<std::string> kns(n_keys), kcs(n_keys), kks(n_keys); std::vector<int32_t> roots(n_keys + 1);
    for (uint32_t i = 0; i < n_keys; i++) { kns[i] = in.bytes(); kcs[i] = in.bytes(); kks[i] = in.bytes(); roots[i] = (int32_t)in.u32(); }
    std::string knb, kcb, kkb; std::vector<uint32_t> kno, kco, kko;
    blob(kns, knb, kno); blob(kcs, kcb, kco); blob(kks, kkb, kko);
    void* k = kl_new();
    if (const char* err = kl_apply(k, 1, (int)n_nodes, (int)n_pr, kn.data(), (int)n_kn, (const uint8_t*)knb.data(), kno.data(), (const uint8_t*)kcb.data(),
                                   kco.data(), (const uint8_t*)kkb.data(), kko.data(), roots.data(), (int)n_keys)) {
        fprintf(stderr, "key table refused: %s\n", err); return 2;
    }
    const uint32_t n_ns = in.u32();
    std::vector<std::string> nsn(n_ns), nsv(n_ns); std::vector<int32_t> nsr(n_ns + 1);
    for (uint32_t i = 0; i < n_ns; i++) { nsn[i] = in.bytes(); nsr[i] = (int32_t)in.u32(); nsv[i] = in.bytes(); }
    std::string nsb, vb; std::vector<uint32_t> nso, vo;
    blob(nsn, nsb, nso); blob(nsv, vb, vo);

    const uint32_t n_blocks = in.u32();
    uint32_t parsed = 0; uint64_t n_tx = 0, lscc = 0;
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t writes_hint = in.u32();
        in.u32();
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
        bd_namespaces(h, (const uint8_t*)nsb.data(), nso.data(), nsr.data(), (int)n_ns);
        const int T = (int)envs.size();
        uint32_t n_rec = 0;
        const int n_end = v13_plan(k, h, env_blob.data(), env_off.data(), T, (int)writes_hint, BD_MODE_V13, &n_rec);
        std::vector<uint8_t> sig_ok(T + n_end + 1, 0), chk(64 * (size_t)T + 1, 0), flags(T + 1, 0), conf(T + 1, 0);
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
                for (int kk = 0; kk < 3; kk++) m.append((const char*)hh->block.data() + segs[6 * q + kk], segs[6 * q + 3 + kk]);
                sha256(m, &chk[64 * (size_t)t + 32 * q]);
            }
        }
        const uint32_t zero = 0;
        int seen = 0;
        v13_decide(k, h, BD_MODE_V13, (const uint8_t*)vb.data(), vo.data(), sig_ok.data(), chk.data(), &zero, 0, (int)n_pr, nullptr, nullptr, nullptr,
                   nullptr, nullptr, 0, flags.data(), conf.data(), &seen);
        printf("flags ");
        for (int t = 0; t < T; t++) printf("%02x", flags[t]);
        printf(" %d\n", seen);
        bd_free(h);
        n_tx += T; lscc += seen != 0;
    }
    kl_free(k);
    fclose(in.f);
    printf("blocks %u parsed %u transactions %llu lscc %llu\n", n_blocks, parsed, (unsigned long long)n_tx, (unsigned long long)lscc);
    return 0;
}
