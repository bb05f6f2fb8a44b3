// schnorr_verify_double_all of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_verify_double_all_cpu.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, a
// batch signed by two keys with schnorr_sign_double_batch passes schnorr_verify_double_all with per-item key pairs, and
// also the signatures of one key under one key pair; one signature's message changed fails it; and a G' off the curve
// throws InvalidPoint.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar sk{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, sk2{{12345, 0, 1, 0}}, g2{{987654321, 3, 0, 0}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            JubJubScalar one{{1, 0, 0, 0}};
            schnorr_verify_double_all(G, G, 1, &one, G, G, G, &one, &one, 1, G, G);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("verify double all mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    Scalar Gp[2];
    fixed_base(g2, G, Gp, e);   // G' = [g2] G, a point of the prime-order subgroup
    // a batch signed by two keys, alternating
    const size_t n = 60;
    Scalar PK[2], PKp[2], PK2[2], PK2p[2];
    fixed_base(sk, G, PK, e);
    fixed_base(sk, Gp, PKp, e);
    fixed_base(sk2, G, PK2, e);
    fixed_base(sk2, Gp, PK2p, e);
    std::vector<JubJubScalar> keys(n), r(n), w(n), wp(n);
    std::vector<Scalar> msg(n), pks(2 * n), pkps(2 * n);
    for (size_t i = 0; i < n; ++i) {
        keys[i] = (i % 2) ? sk2 : sk;
        r[i] = JubJubScalar{{3 * i + 1, i, 0, i << 20}};
        w[i] = JubJubScalar{{0x9e3779b97f4a7c15ULL * (i + 1), 0x632be59bd9b4e019ULL ^ i, 0, 0}};
        wp[i] = JubJubScalar{{0xbf58476d1ce4e5b9ULL * (i + 3), 0x94d049bb133111ebULL + i, 0, 0}};
        msg[i] = Scalar{{i * i + 1, i, 0, 0}};
        const Scalar* pk = (i % 2) ? PK2 : PK;
        const Scalar* pkp = (i % 2) ? PK2p : PKp;
        pks[2 * i] = pk[0], pks[2 * i + 1] = pk[1];
        pkps[2 * i] = pkp[0], pkps[2 * i + 1] = pkp[1];
    }
    std::vector<Scalar> R, Rp;
    std::vector<uint8_t> ok;
    const auto u = schnorr_sign_double_batch(keys.data(), n, r.data(), msg.data(), n, G, Gp, R, Rp, ok, e);
    size_t bad = 9;
    if (!schnorr_verify_double_all(pks.data(), pkps.data(), n, u.data(), R.data(), Rp.data(), msg.data(), w.data(),
                                   wp.data(), n, G, Gp, &bad, e) ||
        bad != 0)
        return 3;
    // one key for the batch
    const auto u1 = schnorr_sign_double_batch(&sk, 1, r.data(), msg.data(), n, G, Gp, R, Rp, ok, e);
    if (!schnorr_verify_double_all(PK, PKp, 1, u1.data(), R.data(), Rp.data(), msg.data(), w.data(), wp.data(), n, G, Gp,
                                   &bad, e) ||
        bad != 0)
        return 4;
    msg[17].l[0] ^= 1;
    if (schnorr_verify_double_all(PK, PKp, 1, u1.data(), R.data(), Rp.data(), msg.data(), w.data(), wp.data(), n, G, Gp,
                                  &bad, e) ||
        bad != 0)
        return 5;
    try {
        Scalar off[2] = {Gp[0], Gp[1]};
        off[1].l[0] ^= 1;
        schnorr_verify_double_all(PK, PKp, 1, u1.data(), R.data(), Rp.data(), msg.data(), w.data(), wp.data(), n, G, off,
                                  nullptr, e);
        return 6;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 7;
    }
    std::puts("verify double all mirror ok (GPU)");
    return 0;
}
