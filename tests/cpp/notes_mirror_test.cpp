// value_commit[_batch] / note_create[_batch] / note_open[_batch] of the C++ mirror (include/poseidon252_b200.hpp) against
// the C ABI.  Built and run by tests/test_notes_cpu.py.  Without a GPU the default engine cannot be created (no CPU
// fallback); with one, G' = [k] G, notes created by note_create_batch for the wallet (A, B) = ([a] G, [b] G) have the
// commitments of value_commit_batch and the note keys of stealth_address, open under a with their (v, blinder) and under
// no other key, the single-item calls agree with the batch ones, and the single-item calls throw InvalidPoint for a
// blinder >= r_J and DecryptionFailed for a note whose commitment does not match.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar k{{0x9e3779b97f4a7c15ULL, 11, 0, 0x0100000000000000ULL}};
    const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Scalar C[2];
            value_commit(5, k, G, G, C);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("notes mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar Gp[2], A[2], B[2];
    fixed_base(k, G, Gp, e);
    const JubJubScalar a{{0xabcdefULL, 3, 0, 0x0200000000000000ULL}}, b{{999, 5, 0, 0}};
    fixed_base(a, G, A, e);
    fixed_base(b, G, B, e);
    const size_t n = 6;
    std::vector<JubJubScalar> r(n), blinder(n);
    std::vector<uint64_t> value(n);
    std::vector<Scalar> nonce(n);
    for (size_t i = 0; i < n; ++i) {
        r[i] = JubJubScalar{{5 * i + 3, i, 0, i << 24}};
        blinder[i] = JubJubScalar{{0x1234567 * (i + 1), i, 7, 0}};
        value[i] = 0xfffffffffffffff0ULL + i;   // carries through every digit
        nonce[i] = Scalar{{i, 0, 0, 0}};
    }
    std::vector<uint8_t> ok;
    const auto C0 = value_commit_batch(value.data(), blinder.data(), n, G, Gp, ok, nullptr, e);
    std::vector<Scalar> R, pk, C, cipher;
    size_t bad = 9;
    ok = note_create_batch(r.data(), value.data(), blinder.data(), nonce.data(), n, G, Gp, A, B, 1, R, pk, C, cipher, &bad, e);
    if (bad != 0 || std::memcmp(C.data(), C0.data(), C.size() * sizeof(Scalar))) return 3;
    for (size_t i = 0; i < n; ++i) {
        Scalar Ri[2], pki[2];
        stealth_address(r[i], G, A, B, Ri, pki, e);
        if (std::memcmp(Ri, &R[2 * i], sizeof Ri) || std::memcmp(pki, &pk[2 * i], sizeof pki)) return 4;
    }
    std::vector<JubJubScalar> b_out;
    size_t failed = 9;
    const auto v_out = note_open_batch(&a, 1, R.data(), nonce.data(), cipher.data(), C.data(), n, G, Gp, b_out, ok, &failed, e);
    if (failed != 0 || v_out != value || std::memcmp(b_out.data(), blinder.data(), n * sizeof(JubJubScalar))) return 5;
    note_open_batch(&b, 1, R.data(), nonce.data(), cipher.data(), C.data(), n, G, Gp, b_out, ok, &failed, e);
    if (failed != n) return 6;                                      // another key opens nothing
    Scalar C1[2];
    value_commit(value[2], blinder[2], G, Gp, C1, e);
    if (std::memcmp(C1, &C[4], sizeof C1)) return 7;
    const Scalar R1[2] = {R[2], R[3]}, Cn[2] = {C[2], C[3]}, Cm[2] = {C[4], C[5]};
    const Scalar ci[3] = {cipher[3], cipher[4], cipher[5]};
    JubJubScalar bo;
    if (note_open(a, R1, nonce[1], ci, Cn, G, Gp, bo, e) != value[1] || std::memcmp(&bo, &blinder[1], sizeof bo)) return 8;
    try {
        note_open(a, R1, nonce[1], ci, Cm, G, Gp, bo, e);         // another note's commitment
        return 9;
    } catch (const Error& err) {
        if (!err.is_decryption_failed()) return 10;
    }
    try {
        value_commit(1, too_big, G, Gp, C1, e);
        return 11;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 12;
    }
    std::puts("notes mirror ok (GPU)");
    return 0;
}
