// Hash::finalize_batch of the C++ mirror (include/poseidon252_b200.hpp) against Hash::finalize and the C ABI.  Built and
// run by tests/test_hash_mixed_cpu.py.  The lowest-index invalid hash decides the exception before any device is needed
// (a Merkle arity violation, a zero-length update() chunk); without a GPU a valid batch then throws P252_ERR_NO_DEVICE
// (no CPU fallback).  With one, hashes of every domain with several update() chunks and output lengths equal
// Hash::finalize item by item, and a truncated item equals p252_hash_batch_truncated over its concatenated input.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    std::vector<Scalar> pool(64);
    for (size_t i = 0; i < pool.size(); ++i)
        for (int k = 0; k < 4; ++k) pool[i].l[k] = (uint64_t)(i * 4 + k + 7) * 0x9e3779b97f4a7c15ULL >> 3;   // < p
    std::vector<Hash> bad;
    bad.emplace_back(Domain::Other);
    bad.back().update(pool.data(), 3);
    bad.emplace_back(Domain::Merkle4);
    bad.back().update(pool.data(), 3);                 // arity violation first ...
    bad.emplace_back(Domain::Other);
    bad.back().update(pool.data(), 0);                 // ... wins over the later zero-length chunk
    try {
        Hash::finalize_batch(bad);
        return 1;
    } catch (const Error& e) {
        if (e.code != P252_ERR_IO_PATTERN_VIOLATION) return 2;
    }
    bad.erase(bad.begin() + 1);
    try {
        Hash::finalize_batch(bad);
        return 3;
    } catch (const Error& e) {
        if (e.code != P252_ERR_INVALID_IO_PATTERN) return 4;
    }
    std::vector<Hash> hs;
    std::vector<bool> trunc;
    const Domain doms[4] = {Domain::Merkle4, Domain::Merkle2, Domain::Encryption, Domain::Other};
    for (int i = 0; i < 12; ++i) {
        const Domain d = doms[i % 4];
        hs.emplace_back(d);
        const size_t len = d == Domain::Merkle4 ? 4 : (d == Domain::Merkle2 ? 2 : 1 + (size_t)(i * 5) % 11);
        if (len > 1) hs.back().update(pool.data() + i, len / 2);   // two chunks: the layout does not change the digest
        hs.back().update(pool.data() + i + len / 2, len - len / 2);
        hs.back().output_len(1 + i % 6);               // honoured for Domain::Other only
        trunc.push_back(i % 3 == 1);
    }
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Hash::finalize_batch(hs, trunc);
            return 5;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 6;
        }
        std::puts("hash_mixed mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    const auto got = Hash::finalize_batch(hs, trunc, &e);
    for (size_t i = 0; i < hs.size(); ++i) {
        if (!trunc[i]) {
            const std::vector<Scalar> want = hs[i].finalize();
            if (got[i].size() != want.size() || std::memcmp(got[i].data(), want.data(), want.size() * sizeof(Scalar))) return 7;
            continue;
        }
        const int d = static_cast<int>(doms[i % 4]);
        const size_t len = d == P252_DOMAIN_MERKLE4 ? 4 : (d == P252_DOMAIN_MERKLE2 ? 2 : 1 + (i * 5) % 11);
        const size_t ol = d == P252_DOMAIN_OTHER ? 1 + i % 6 : 1;
        std::vector<Scalar> want(ol);
        check(p252_hash_batch_truncated(e.get(), d, pool.data() + i, 1, len, want.data(), ol, P252_MEM_HOST));
        if (got[i].size() != ol || std::memcmp(got[i].data(), want.data(), ol * sizeof(Scalar))) return 8;
    }
    std::puts("hash_mixed mirror ok");
    return 0;
}
