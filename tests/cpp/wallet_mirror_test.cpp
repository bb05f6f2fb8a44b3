// wallet_scan_batch of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_wallet_cpu.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, notes created
// by note_create_batch for two wallets (A_j, B_j) = ([a_j] G, [b_j] G) are scanned with both keys: each note's owner is
// the wallet it was made for, its nullifier is nullifier_batch's under that key, its opening note_open_batch's, and the
// totals add up the values.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar kp{{0x9e3779b97f4a7c15ULL, 11, 0, 0x0100000000000000ULL}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            const JubJubScalar one{{1, 0, 0, 0}};
            const uint64_t pos = 0;
            wallet_scan_batch(&one, &one, 1, G, G, &pos, G, G, G, 1, G, G);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("wallet mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar Gp[2];
    fixed_base(kp, G, Gp, e);
    const JubJubScalar a[2] = {JubJubScalar{{0xabcdefULL, 3, 0, 0x0200000000000000ULL}}, JubJubScalar{{77, 1, 2, 3}}};
    const JubJubScalar b[2] = {JubJubScalar{{999, 5, 0, 0}}, JubJubScalar{{4242, 0, 9, 0}}};
    const size_t n = 6;
    std::vector<Scalar> R(2 * n), pk(2 * n), C(2 * n), cipher(3 * n), nonce(n);
    std::vector<uint64_t> value(n), pos(n);
    std::vector<JubJubScalar> blinder(n);
    for (size_t i = 0; i < n; ++i) {
        const size_t w = i % 2;
        Scalar A[2], B[2];
        fixed_base(a[w], G, A, e);
        fixed_base(b[w], G, B, e);
        const JubJubScalar r{{5 * i + 3, i, 0, i << 24}};
        blinder[i] = JubJubScalar{{0x1234567 * (i + 1), i, 7, 0}};
        value[i] = 0xfffffffffffffff0ULL + i;
        nonce[i] = Scalar{{i, 0, 0, 0}};
        pos[i] = 1000 + i;
        std::vector<Scalar> Ri, pki, Ci, ci;
        note_create_batch(&r, &value[i], &blinder[i], &nonce[i], 1, G, Gp, A, B, 1, Ri, pki, Ci, ci, nullptr, e);
        std::copy(Ri.begin(), Ri.end(), R.begin() + 2 * i);
        std::copy(pki.begin(), pki.end(), pk.begin() + 2 * i);
        std::copy(Ci.begin(), Ci.end(), C.begin() + 2 * i);
        std::copy(ci.begin(), ci.end(), cipher.begin() + 3 * i);
    }
    const WalletScan w = wallet_scan_batch(a, b, 2, R.data(), pk.data(), pos.data(), nonce.data(), cipher.data(), C.data(), n,
                                           G, Gp, e);
    if (w.n_invalid != 0 || w.n_bad_keys != 0) return 3;
    unsigned __int128 sum[2] = {0, 0};
    for (size_t i = 0; i < n; ++i) {
        const size_t j = i % 2;
        if (w.owner[i] != (int32_t)j || !w.opened[i] || w.value[i] != value[i]) return 4;
        if (std::memcmp(&w.blinder[i], &blinder[i], sizeof(JubJubScalar))) return 5;
        const Scalar Ri[2] = {R[2 * i], R[2 * i + 1]};
        const Scalar nul = nullifier(a[j], b[j], Gp, Ri, pos[i], e);
        if (std::memcmp(&nul, &w.nullifier[i], sizeof(Scalar))) return 6;
        sum[j] += value[i];
    }
    for (size_t j = 0; j < 2; ++j)
        if (w.key_totals[4 * j] != (uint64_t)sum[j] || w.key_totals[4 * j + 1] != (uint64_t)(sum[j] >> 64) ||
            w.key_totals[4 * j + 2] != 3 || w.key_totals[4 * j + 3] != 3)
            return 7;
    std::puts("wallet mirror ok (GPU)");
    return 0;
}
