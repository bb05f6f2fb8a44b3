// nullifier / nullifier_batch of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_nullifier_cpu.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, for notes
// made by stealth_address to the wallet (A, B) = ([a] G, [b] G), [note_sk] G is the note's key, so with G' = G the
// nullifier at position pos is Hash::digest(Other, [note_pk.u, note_pk.v, pos]); the batch call agrees with the single
// one, another wallet's key gives other nullifiers, and nullifier() throws InvalidPoint for an a >= r_J.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const Scalar zero{{0, 0, 0, 0}};
    const Scalar one{{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
    const JubJubScalar a{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, b{{12345, 0, 1, 0}};
    const JubJubScalar a2{{0xabcdefULL, 3, 0, 0x0200000000000000ULL}}, b2{{999, 5, 0, 0}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            nullifier(a, b, G, G, 0);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("nullifier mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar A[2], B[2];
    fixed_base(a, G, A, e);
    fixed_base(b, G, B, e);
    const size_t n = 8;
    std::vector<Scalar> R(2 * n), pk(2 * n);
    std::vector<uint64_t> pos(n);
    for (size_t i = 0; i < n; ++i) {
        const JubJubScalar r{{5 * i + 3, i, 0, i << 24}};
        Scalar Ri[2], pki[2];
        stealth_address(r, G, A, B, Ri, pki, e);
        R[2 * i] = Ri[0], R[2 * i + 1] = Ri[1], pk[2 * i] = pki[0], pk[2 * i + 1] = pki[1];
        pos[i] = i % 2;
    }
    std::vector<uint8_t> ok;
    size_t bad = 9;
    const auto nul = nullifier_batch(&a, &b, 1, G, R.data(), pos.data(), n, ok, &bad, e);
    if (bad != 0) return 3;
    for (size_t i = 0; i < n; ++i) {
        if (!ok[i]) return 4;
        const auto want = Hash::digest(Domain::Other, {pk[2 * i], pk[2 * i + 1], pos[i] ? one : zero}, &e);
        if (std::memcmp(&nul[i], &want[0], sizeof(Scalar))) return 5;
    }
    const Scalar R0[2] = {R[0], R[1]};
    const Scalar one_note = nullifier(a, b, G, R0, pos[0], e);
    if (std::memcmp(&one_note, &nul[0], sizeof(Scalar))) return 6;
    const Scalar other = nullifier(a2, b2, G, R0, pos[0], e);
    if (!std::memcmp(&other, &nul[0], sizeof(Scalar))) return 7;
    try {
        const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
        nullifier(too_big, b, G, R0, 0, e);
        return 8;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 9;
    }
    std::puts("nullifier mirror ok (GPU)");
    return 0;
}
