// The C++ CompactTree (include/poseidon252_b200.hpp) against the C ABI.  Built and run by tests/test_ctree_bindings.py
// (the loud failure without a GPU, and the GPU run).  With a GPU: inserts value i at position i * 0x9e3779b97f4a7c15
// (mod 2^64) for i < 300 into an arity-4, height-32 tree, removes every third of them, checks size / contains, an
// opening, a refused opening and a refused over-capacity batch, prints the root.
#include <cstdio>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            CompactTree t(4, 32, 1000);
            return 3;   // no CPU fallback: the default engine cannot be created
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 4;
        }
        std::puts("ctree mirror ok (no GPU)");
        return 0;
    }
    std::vector<Scalar> vals;
    std::vector<uint64_t> pos, gone;
    for (uint64_t i = 0; i < 300; ++i) {
        vals.push_back(Scalar{{1000 + i, i, 0, 0}});
        pos.push_back(i * 0x9e3779b97f4a7c15ull);
        if (i % 3 == 0) gone.push_back(pos.back());
    }
    CompactTree t(4, 32, 300);
    t.insert(pos, vals);
    t.remove(gone);
    if (t.size() != 200 || t.contains(pos[0]) || !t.contains(pos[1]) || t.contains(pos[1] + 1)) return 6;
    Opening o = t.opening(pos[5]);
    if (!o.verify(vals[5]) || o.verify(vals[4])) return 7;
    try {
        t.opening(pos[3]);                             // removed: refused
        return 8;
    } catch (const Error& e) {
        if (e.code != P252_ERR_INVALID_ARGUMENT) return 9;
    }
    std::vector<uint64_t> fresh;
    for (uint64_t k = 1; k <= 101; ++k) fresh.push_back(k);
    try {
        t.insert(fresh, std::vector<Scalar>(101, vals[0]));   // 301 present positions > max_leaves: refused, nothing modified
        return 10;
    } catch (const Error& e) {
        if (e.code != P252_ERR_INVALID_ARGUMENT || t.size() != 200) return 11;
    }
    const Scalar& r = t.root();
    std::printf("root %llu %llu %llu %llu\n", (unsigned long long)r.l[0], (unsigned long long)r.l[1],
                (unsigned long long)r.l[2], (unsigned long long)r.l[3]);
    return 0;
}
