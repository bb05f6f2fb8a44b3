// stealth_address / stealth_address_batch / owns / stealth_owns_batch of the C++ mirror (include/poseidon252_b200.hpp)
// against the C ABI.  Built and run by tests/test_stealth_cpu.py.  Without a GPU the default engine cannot be created (no
// CPU fallback); with one, a note made by stealth_address is owned by its receiver and not by another view key, the
// batch scan finds exactly one receiver's notes among two receivers', R equals fixed_base_batch, and owns() throws
// InvalidPoint for a view key >= r_J.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar a{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, b{{12345, 0, 1, 0}};
    const JubJubScalar a2{{0xabcdefULL, 3, 0, 0x0200000000000000ULL}}, b2{{999, 5, 0, 0}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Scalar R[2], pk[2];
            stealth_address(a, G, G, G, R, pk);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("stealth mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar A[2], B[2], A2[2], B2[2];
    fixed_base(a, G, A, e);
    fixed_base(b, G, B, e);
    fixed_base(a2, G, A2, e);
    fixed_base(b2, G, B2, e);
    // one note
    const JubJubScalar r0{{77, 1, 2, 3}};
    Scalar R0[2], pk0[2];
    stealth_address(r0, G, A, B, R0, pk0, e);
    if (!owns(a, B, G, R0, pk0, e)) return 3;
    if (owns(a2, B2, G, R0, pk0, e) || owns(a2, B, G, R0, pk0, e)) return 4;
    // a batch to two receivers, alternating: receiver 1 owns exactly the even notes
    const size_t n = 40;
    std::vector<JubJubScalar> r(n);
    std::vector<Scalar> As(2 * n), Bs(2 * n);
    for (size_t i = 0; i < n; ++i) {
        r[i] = JubJubScalar{{3 * i + 1, i, 0, i << 20}};
        const Scalar* pa = (i % 2) ? A2 : A;
        const Scalar* pb = (i % 2) ? B2 : B;
        As[2 * i] = pa[0], As[2 * i + 1] = pa[1], Bs[2 * i] = pb[0], Bs[2 * i + 1] = pb[1];
    }
    std::vector<Scalar> R;
    std::vector<uint8_t> ok;
    const auto pk = stealth_address_batch(r.data(), n, G, As.data(), Bs.data(), n, R, ok, e);
    for (auto v : ok)
        if (!v) return 5;
    std::vector<uint8_t> ok2;
    const auto Rf = fixed_base_batch(r.data(), n, G, ok2, e);
    if (std::memcmp(R.data(), Rf.data(), R.size() * sizeof(Scalar))) return 6;
    size_t mine = 0, bad = 9;
    const auto owned = stealth_owns_batch(a, B, G, R.data(), pk.data(), n, &mine, &bad, e);
    if (mine != n / 2 || bad != 0) return 7;
    for (size_t i = 0; i < n; ++i)
        if (owned[i] != (i % 2 == 0 ? 1 : 0)) return 8;
    try {
        const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
        owns(too_big, B, G, R0, pk0, e);
        return 9;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 10;
    }
    std::puts("stealth mirror ok (GPU)");
    return 0;
}
