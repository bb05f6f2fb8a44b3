// schnorr_sign / schnorr_sign_batch / schnorr_verify / schnorr_verify_batch of the C++ mirror
// (include/poseidon252_b200.hpp) against the C ABI.  Built and run by tests/test_schnorr_cpu.py.  Without a GPU the default
// engine cannot be created (no CPU fallback); with one, a signature made by schnorr_sign verifies under its key and not
// under another, a batch signed by two keys verifies under per-item keys, R equals fixed_base_batch of the nonces, and
// schnorr_sign throws InvalidPoint for a key >= r_J.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar sk{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, sk2{{12345, 0, 1, 0}};
    const Scalar m0{{42, 0, 0, 0}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            JubJubScalar u;
            Scalar R[2];
            schnorr_sign(sk, sk2, m0, G, u, R);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("schnorr mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar PK[2], PK2[2];
    fixed_base(sk, G, PK, e);
    fixed_base(sk2, G, PK2, e);
    // one signature
    const JubJubScalar r0{{77, 1, 2, 3}};
    JubJubScalar u0;
    Scalar R0[2];
    schnorr_sign(sk, r0, m0, G, u0, R0, e);
    if (!schnorr_verify(PK, u0, R0, m0, G, e)) return 3;
    if (schnorr_verify(PK2, u0, R0, m0, G, e)) return 4;
    // a batch signed by two keys, alternating
    const size_t n = 40;
    std::vector<JubJubScalar> keys(n), r(n);
    std::vector<Scalar> msg(n), pks(2 * n);
    for (size_t i = 0; i < n; ++i) {
        keys[i] = (i % 2) ? sk2 : sk;
        r[i] = JubJubScalar{{3 * i + 1, i, 0, i << 20}};
        msg[i] = Scalar{{i * i + 1, i, 0, 0}};
        const Scalar* pk = (i % 2) ? PK2 : PK;
        pks[2 * i] = pk[0], pks[2 * i + 1] = pk[1];
    }
    std::vector<Scalar> R;
    std::vector<uint8_t> ok;
    const auto u = schnorr_sign_batch(keys.data(), n, r.data(), msg.data(), n, G, R, ok, e);
    for (auto v : ok)
        if (!v) return 5;
    std::vector<uint8_t> ok2;
    const auto Rf = fixed_base_batch(r.data(), n, G, ok2, e);
    if (std::memcmp(R.data(), Rf.data(), R.size() * sizeof(Scalar))) return 6;
    size_t good = 0, bad = 9;
    auto verified = schnorr_verify_batch(pks.data(), n, u.data(), R.data(), msg.data(), n, G, &good, &bad, e);
    if (good != n || bad != 0) return 7;
    // under the first key alone exactly the even signatures verify
    verified = schnorr_verify_batch(PK, 1, u.data(), R.data(), msg.data(), n, G, &good, &bad, e);
    if (good != n / 2 || bad != 0) return 8;
    for (size_t i = 0; i < n; ++i)
        if (verified[i] != (i % 2 == 0 ? 1 : 0)) return 9;
    try {
        const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
        JubJubScalar u1;
        Scalar R1[2];
        schnorr_sign(too_big, r0, m0, G, u1, R1, e);
        return 10;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 11;
    }
    std::puts("schnorr mirror ok (GPU)");
    return 0;
}
