// The C++ SparseTree (include/poseidon252_b200.hpp) against the C ABI.  Built and run by tests/test_smtree_bindings.py
// (the loud failure without a GPU) and tests/test_gpu_smtree.py.  With a GPU: reads values as "l0 l1 l2 l3" lines on
// stdin (at least 300; synthetic ones without input), inserts value i at position 7 * i + 3 for i < 300, removes every
// third of those positions, checks len / contains, an opening and a refused update, prints the root.
#include <cstdio>
#include <iostream>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            SparseTree t(4, 8, 5000);
            return 3;   // no CPU fallback: the default engine cannot be created
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 4;
        }
        std::puts("smtree mirror ok (no GPU)");
        return 0;
    }
    std::vector<Scalar> vals;
    Scalar s{};
    while (std::cin >> s.l[0] >> s.l[1] >> s.l[2] >> s.l[3]) vals.push_back(s);
    for (uint64_t i = vals.size(); i < 300; ++i) vals.push_back(Scalar{{1000 + i, i, 0, 0}});   // no input: synthetic
    vals.resize(300);
    std::vector<uint64_t> pos, gone;
    for (uint64_t i = 0; i < 300; ++i) pos.push_back(7 * i + 3);
    for (uint64_t i = 0; i < 300; i += 3) gone.push_back(7 * i + 3);
    SparseTree t(4, 8, 5000);
    t.insert(pos, vals);
    t.remove(gone);
    if (t.size() != 200 || t.contains(3) || !t.contains(10) || t.contains(11)) return 6;
    Opening o = t.opening(7 * 5 + 3);
    if (!o.verify(vals[5]) || o.verify(vals[4])) return 7;
    try {
        t.opening(3);                                  // removed: refused
        return 8;
    } catch (const Error& e) {
        if (e.code != P252_ERR_INVALID_ARGUMENT) return 9;
    }
    try {
        t.insert({5000}, {vals[0]});                   // beyond the capacity: refused, nothing modified
        return 10;
    } catch (const Error& e) {
        if (e.code != P252_ERR_INVALID_ARGUMENT) return 11;
    }
    const Scalar& r = t.root();
    std::printf("root %llu %llu %llu %llu\n", (unsigned long long)r.l[0], (unsigned long long)r.l[1],
                (unsigned long long)r.l[2], (unsigned long long)r.l[3]);
    return 0;
}
