// Hash::digest_batch_varlen of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_varlen_bindings.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, every
// length 1..40 in one call equals Hash::digest per item, and an empty item throws InvalidIOPattern.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    std::vector<std::vector<Scalar>> inputs;
    for (uint64_t len = 40; len >= 1; --len) {
        std::vector<Scalar> in;
        for (uint64_t j = 0; j < len; ++j) in.push_back(Scalar{{len * 100 + j, j, 0, 0}});
        inputs.push_back(in);
    }
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Hash::digest_batch_varlen(Domain::Other, inputs, 3);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("varlen mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    const auto got = Hash::digest_batch_varlen(Domain::Other, inputs, 3, e);
    if (got.size() != inputs.size()) return 3;
    for (size_t i = 0; i < inputs.size(); ++i) {
        Hash h(Domain::Other, &e);
        h.output_len(3);
        h.update(inputs[i]);
        const auto want = h.finalize();
        if (got[i].size() != 3 || std::memcmp(got[i].data(), want.data(), 3 * sizeof(Scalar))) return 4;
    }
    inputs[7].clear();
    try {
        Hash::digest_batch_varlen(Domain::Other, inputs, 1, e);
        return 5;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_IO_PATTERN) return 6;
    }
    std::puts("varlen mirror ok (GPU)");
    return 0;
}
