// hash_to_scalar_batch / scalars_from_bytes_wide of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.
// Built and run by tests/test_hash_to_scalar_cpu.py.  Without a GPU the default engine cannot be created (no CPU
// fallback); with one, messages of lengths around the 128-byte block edges hash to what the host's p252_hash_to_scalar
// gives, from_bytes_wide of 1 and of 2^256 gives their Montgomery forms, and a message longer than
// P252_HASH_TO_SCALAR_MAX_LEN throws.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    std::vector<std::vector<uint8_t>> msgs;
    for (size_t len : {0, 1, 63, 64, 127, 128, 129, 255, 256, 257, 1000}) {
        std::vector<uint8_t> m(len);
        for (size_t i = 0; i < len; ++i) m[i] = (uint8_t)(i * 131 + len);
        msgs.push_back(m);
    }
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            hash_to_scalar_batch(msgs);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("hash_to_scalar mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    const std::vector<Scalar> got = hash_to_scalar_batch(msgs, e);
    if (got.size() != msgs.size()) return 3;
    for (size_t i = 0; i < msgs.size(); ++i) {
        Scalar want;
        check(p252_hash_to_scalar(msgs[i].data(), msgs[i].size(), &want));
        if (std::memcmp(&want, &got[i], sizeof want)) return 4;
    }
    // from_bytes_wide: (lo + hi 2^256) mod p; lo = 1, hi = 0 is the scalar 1 (Montgomery form R mod p)
    uint8_t rows[2][64] = {};
    rows[0][0] = 1;
    rows[1][32] = 1;                                    // 2^256 mod p = R mod p, in Montgomery form R^2 mod p
    const std::vector<Scalar> w = scalars_from_bytes_wide(&rows[0][0], 2, e);
    const Scalar one{{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
    const Scalar r2{{0xc999e990f3f29c6dULL, 0x2b6cedcb87925c23ULL, 0x05d314967254398fULL, 0x0748d9d99f59ff11ULL}};
    if (std::memcmp(&w[0], &one, sizeof one) || std::memcmp(&w[1], &r2, sizeof r2)) return 5;
    std::vector<std::vector<uint8_t>> too_long(1, std::vector<uint8_t>(P252_HASH_TO_SCALAR_MAX_LEN + 1));
    try {
        hash_to_scalar_batch(too_long, e);
        return 6;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_ARGUMENT) return 7;
    }
    std::puts("hash_to_scalar mirror ok");
    return 0;
}
