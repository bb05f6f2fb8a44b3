// point_from_bytes / points_from_bytes_batch / point_to_bytes / points_to_bytes_batch of the C++ mirror
// (include/poseidon252_b200.hpp) against the C ABI.  Built and run by tests/test_points_cpu.py.  Without a GPU the default
// engine cannot be created (no CPU fallback); with one, the encodings of a batch of fixed_base_batch points decode back to
// the same points, an all-0xff encoding and an off-curve point throw InvalidPoint, and the batch forms count them.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            uint8_t b[32];
            point_to_bytes(G, b);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("points mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    // one point
    uint8_t gb[32];
    point_to_bytes(G, gb, e);
    Scalar g2[2];
    point_from_bytes(gb, g2, e);
    if (std::memcmp(g2, G, sizeof G)) return 3;
    // a batch of [k] G
    const size_t n = 50;
    std::vector<JubJubScalar> ks(n);
    for (size_t i = 0; i < n; ++i) ks[i] = JubJubScalar{{7 * i + 1, i, i << 9, 0}};
    std::vector<uint8_t> ok;
    const auto pts = fixed_base_batch(ks.data(), n, G, ok, e);
    size_t bad = 9;
    const auto bytes = points_to_bytes_batch(pts.data(), n, ok, &bad, e);
    if (bad != 0 || bytes.size() != 32 * n) return 4;
    const auto back = points_from_bytes_batch(bytes.data(), n, ok, &bad, e);
    if (bad != 0 || std::memcmp(back.data(), pts.data(), pts.size() * sizeof(Scalar))) return 5;
    // invalid items
    uint8_t ff[32];
    std::memset(ff, 0xff, sizeof ff);
    try {
        Scalar uv[2];
        point_from_bytes(ff, uv, e);
        return 6;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 7;
    }
    try {
        const Scalar off[2] = {G[1], G[0]};
        uint8_t b[32];
        point_to_bytes(off, b, e);
        return 8;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 9;
    }
    std::puts("points mirror ok (GPU)");
    return 0;
}
