// schnorr_sign_double[_batch] / schnorr_verify_double[_batch] / note_sign_double_batch of the C++ mirror
// (include/poseidon252_b200.hpp) against the C ABI.  Built and run by tests/test_schnorr_double_cpu.py.  Without a GPU the
// default engine cannot be created (no CPU fallback); with one, G' = [k] G, a key pair ([sk] G, [sk] G') verifies its
// signatures and not another key's, the batch calls agree with the single ones, the note signer's signatures verify under
// (note_pk, pk') for notes made by stealth_address, pk' is the point whose nullifier p252::nullifier computes, and the
// single-item calls throw InvalidPoint for a secret >= r_J.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const Scalar one{{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
    const JubJubScalar k{{0x9e3779b97f4a7c15ULL, 11, 0, 0x0100000000000000ULL}};
    const JubJubScalar sk{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, sk2{{12345, 0, 1, 0}};
    const JubJubScalar too_big{{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            JubJubScalar u;
            Scalar R[2], Rp[2];
            schnorr_sign_double(sk, sk2, one, G, G, u, R, Rp);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("schnorr double mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar Gp[2], PK[2], PKp[2];
    fixed_base(k, G, Gp, e);
    fixed_base(sk, G, PK, e);
    fixed_base(sk, Gp, PKp, e);
    const size_t n = 6;
    std::vector<JubJubScalar> r(n);
    std::vector<Scalar> msg(n);
    for (size_t i = 0; i < n; ++i) r[i] = JubJubScalar{{7 * i + 1, i, 3, i << 20}}, msg[i] = Scalar{{i, 0, 0, 0}};
    std::vector<Scalar> R, Rp;
    std::vector<uint8_t> ok;
    const auto u = schnorr_sign_double_batch(&sk, 1, r.data(), msg.data(), n, G, Gp, R, Rp, ok, e);
    for (size_t i = 0; i < n; ++i)
        if (!ok[i]) return 3;
    size_t nver = 0, bad = 9;
    auto ver = schnorr_verify_double_batch(PK, PKp, 1, u.data(), R.data(), Rp.data(), msg.data(), n, G, Gp, &nver, &bad, e);
    if (nver != n || bad != 0) return 4;
    JubJubScalar u0;
    Scalar R0[2], Rp0[2];
    schnorr_sign_double(sk, r[0], msg[0], G, Gp, u0, R0, Rp0, e);
    if (std::memcmp(&u0, &u[0], sizeof u0) || std::memcmp(R0, R.data(), sizeof R0) || std::memcmp(Rp0, Rp.data(), sizeof Rp0))
        return 5;
    if (!schnorr_verify_double(PK, PKp, u0, R0, Rp0, msg[0], G, Gp, e)) return 6;
    if (schnorr_verify_double(PK, PK, u0, R0, Rp0, msg[0], G, Gp, e)) return 7;          // PK' replaced by PK
    if (schnorr_verify_double(PK, PKp, u0, Rp0, R0, msg[0], G, Gp, e)) return 8;         // R and R' swapped
    try {
        schnorr_sign_double(too_big, r[0], msg[0], G, Gp, u0, R0, Rp0, e);
        return 9;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 10;
    }
    // spending notes made by stealth_address to the wallet (A, B) = ([a] G, [b] G)
    const JubJubScalar a{{0xabcdefULL, 3, 0, 0x0200000000000000ULL}}, b{{999, 5, 0, 0}};
    Scalar A[2], B[2];
    fixed_base(a, G, A, e);
    fixed_base(b, G, B, e);
    std::vector<Scalar> note_R(2 * n), note_pk(2 * n);
    for (size_t i = 0; i < n; ++i) {
        Scalar Ri[2], pki[2];
        stealth_address(JubJubScalar{{5 * i + 3, i, 0, i << 24}}, G, A, B, Ri, pki, e);
        note_R[2 * i] = Ri[0], note_R[2 * i + 1] = Ri[1], note_pk[2 * i] = pki[0], note_pk[2 * i + 1] = pki[1];
    }
    std::vector<Scalar> pkp;
    bad = 9;
    const auto un = note_sign_double_batch(&a, &b, 1, note_R.data(), r.data(), msg.data(), n, G, Gp, R, Rp, pkp, ok, &bad, e);
    if (bad != 0) return 11;
    ver = schnorr_verify_double_batch(note_pk.data(), pkp.data(), n, un.data(), R.data(), Rp.data(), msg.data(), n, G, Gp,
                                      &nver, &bad, e);
    if (nver != n || bad != 0) return 12;
    const Scalar Rn0[2] = {note_R[0], note_R[1]};
    const Scalar nul = nullifier(a, b, Gp, Rn0, 1, e);
    const auto want = Hash::digest(Domain::Other, {pkp[0], pkp[1], one}, &e);
    if (std::memcmp(&nul, &want[0], sizeof(Scalar))) return 13;
    const JubJubScalar a2{{0xabcdeeULL, 3, 0, 0x0200000000000000ULL}};
    const auto u2 = note_sign_double_batch(&a2, &b, 1, note_R.data(), r.data(), msg.data(), n, G, Gp, R, Rp, pkp, ok, &bad, e);
    ver = schnorr_verify_double_batch(note_pk.data(), pkp.data(), n, u2.data(), R.data(), Rp.data(), msg.data(), n, G, Gp,
                                      &nver, &bad, e);
    if (nver != 0) return 14;                                       // another wallet's key does not sign for these notes
    std::puts("schnorr double mirror ok (GPU)");
    return 0;
}
