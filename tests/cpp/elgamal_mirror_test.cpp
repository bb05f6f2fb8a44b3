// elgamal_* / note_sender_* of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_elgamal_cpu.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, messages
// encrypted under PK = [sk] G decrypt to themselves under sk and to other points under another key, and the sender of
// notes made by stealth_address to the wallet (A, B) = ([a] G, [b] G) comes back under (a, b) and not under another
// wallet's key.
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
            std::vector<Scalar> c1, c2;
            elgamal_encrypt_batch(G, 1, G, &a, 1, G, c1, c2);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("elgamal mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar A[2], B[2];
    fixed_base(a, G, A, e);
    fixed_base(b, G, B, e);
    const size_t n = 8;
    std::vector<Scalar> msg(2 * n), R(2 * n), pk(2 * n);
    std::vector<JubJubScalar> r(n), blinder(2 * n);
    for (size_t i = 0; i < n; ++i) {
        const JubJubScalar k{{3 * i + 1, i, 0, i << 20}};
        Scalar Mi[2], Ri[2], pki[2];
        fixed_base(k, G, Mi, e);
        stealth_address(k, G, A, B, Ri, pki, e);
        msg[2 * i] = Mi[0], msg[2 * i + 1] = Mi[1];
        R[2 * i] = Ri[0], R[2 * i + 1] = Ri[1], pk[2 * i] = pki[0], pk[2 * i + 1] = pki[1];
        r[i] = JubJubScalar{{7 * i + 5, 0, i, 0}};
        blinder[2 * i] = JubJubScalar{{11 * i + 2, 1, 0, 0}}, blinder[2 * i + 1] = JubJubScalar{{13 * i + 9, 0, 2, 0}};
    }
    std::vector<Scalar> c1, c2;
    size_t bad = 9;
    auto ok = elgamal_encrypt_batch(A, 1, msg.data(), r.data(), n, G, c1, c2, &bad, e);
    if (bad != 0) return 3;
    const auto back = elgamal_decrypt_batch(&a, 1, c1.data(), c2.data(), n, ok, &bad, e);
    if (bad != 0 || std::memcmp(back.data(), msg.data(), msg.size() * sizeof(Scalar))) return 4;
    const auto wrong = elgamal_decrypt_batch(&a2, 1, c1.data(), c2.data(), n, ok, &bad, e);
    if (bad != 0 || ok[0] != 1 || !std::memcmp(wrong.data(), msg.data(), 2 * sizeof(Scalar))) return 5;   // not authenticated
    std::vector<Scalar> enc, gotA, gotB;
    ok = note_sender_encrypt_batch(pk.data(), A, B, 1, blinder.data(), n, G, enc, &bad, e);
    if (bad != 0) return 6;
    ok = note_sender_decrypt_batch(&a, &b, 1, R.data(), pk.data(), enc.data(), n, G, gotA, gotB, &bad, e);
    if (bad != 0) return 7;
    for (size_t i = 0; i < n; ++i)
        if (!ok[i] || std::memcmp(&gotA[2 * i], A, sizeof A) || std::memcmp(&gotB[2 * i], B, sizeof B)) return 8;
    ok = note_sender_decrypt_batch(&a2, &b2, 1, R.data(), pk.data(), enc.data(), n, G, gotA, gotB, &bad, e);
    if (bad != n) return 9;
    for (size_t i = 0; i < n; ++i)
        if (ok[i]) return 10;
    std::puts("elgamal mirror ok (GPU)");
    return 0;
}
