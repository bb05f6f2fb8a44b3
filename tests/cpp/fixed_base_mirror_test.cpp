// fixed_base / fixed_base_batch / encrypt_batch_ephemeral of the C++ mirror (include/poseidon252_b200.hpp) against the C
// ABI.  Built and run by tests/test_fixed_base_cpu.py.  Without a GPU the default engine cannot be created (no CPU
// fallback); with one, the fixed-base results equal dhke_batch on the same base, the sender's fused call round-trips
// through the receiver's decrypt_batch_dhke, and fixed_base() throws InvalidPoint for a secret >= r_J.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar a{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Scalar out[2];
            fixed_base(a, G, out);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("fixed_base mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    const size_t n = 40, L = 2;
    std::vector<JubJubScalar> r(n);
    std::vector<Scalar> msg(n * L), nonce(n);
    for (size_t i = 0; i < n; ++i) {
        r[i] = JubJubScalar{{3 * i + 1, i, 0, i << 20}};
        nonce[i] = Scalar{{i, 1, 0, 0}};
        for (size_t k = 0; k < L; ++k) msg[i * L + k] = Scalar{{i * 10 + k, 2, 0, 0}};
    }
    Scalar pk[2];
    fixed_base(a, G, pk, e);
    std::vector<uint8_t> ok;
    const auto R = fixed_base_batch(r.data(), n, G, ok, e);
    const auto Rd = dhke_batch(r.data(), n, G, 1, n, ok, e);
    if (std::memcmp(R.data(), Rd.data(), R.size() * sizeof(Scalar))) return 3;
    std::vector<Scalar> R2;
    const auto cipher = encrypt_batch_ephemeral(msg.data(), n, L, r.data(), G, pk, 1, nonce.data(), R2, ok, e);
    for (auto v : ok)
        if (!v) return 4;
    if (std::memcmp(R2.data(), R.data(), R.size() * sizeof(Scalar))) return 5;
    const auto back = decrypt_batch_dhke(cipher.data(), n, L, &a, 1, R2.data(), n, nonce.data(), ok, e);
    for (auto v : ok)
        if (!v) return 6;
    if (std::memcmp(back.data(), msg.data(), msg.size() * sizeof(Scalar))) return 7;
    try {
        const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
        Scalar out[2];
        fixed_base(too_big, G, out, e);
        return 8;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 9;
    }
    std::puts("fixed_base mirror ok (GPU)");
    return 0;
}
