// jubjub_msm / schnorr_verify_all of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built and run by
// tests/test_msm_cpu.py.  Without a GPU the default engine cannot be created (no CPU fallback); with one, the MSM of
// points [k_i] G equals fixed_base of sum s_i k_i, a batch signed by two keys passes schnorr_verify_all with per-item keys
// and fails it with one signature's message changed, and a base off the curve throws InvalidPoint.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    const Scalar G[2] = {Scalar{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                         Scalar{{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
    const JubJubScalar sk{{0xfeedfacecafebeefULL, 7, 9, 0x0123456789abcdefULL}}, sk2{{12345, 0, 1, 0}};
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            Scalar out[2];
            jubjub_msm(&sk, G, 1, out);
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("msm mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    // sum s_i [k_i] G with small k_i, s_i: equal to [sum s_i k_i] G
    const size_t n = 50;
    std::vector<JubJubScalar> k(n), s(n);
    uint64_t total = 0;
    for (size_t i = 0; i < n; ++i) {
        k[i] = JubJubScalar{{1000 + 7 * i, 0, 0, 0}};
        s[i] = JubJubScalar{{3 * i + 1, 0, 0, 0}};
        total += (1000 + 7 * i) * (3 * i + 1);
    }
    std::vector<uint8_t> ok;
    const auto pts = fixed_base_batch(k.data(), n, G, ok, e);
    Scalar got[2], want[2];
    size_t bad = 9;
    jubjub_msm(s.data(), pts.data(), n, got, &bad, e);
    fixed_base(JubJubScalar{{total, 0, 0, 0}}, G, want, e);
    if (bad != 0 || std::memcmp(got, want, sizeof got)) return 3;
    // a batch signed by two keys, alternating
    Scalar PK[2], PK2[2];
    fixed_base(sk, G, PK, e);
    fixed_base(sk2, G, PK2, e);
    std::vector<JubJubScalar> keys(n), r(n), w(n);
    std::vector<Scalar> msg(n), pks(2 * n);
    for (size_t i = 0; i < n; ++i) {
        keys[i] = (i % 2) ? sk2 : sk;
        r[i] = JubJubScalar{{3 * i + 1, i, 0, i << 20}};
        w[i] = JubJubScalar{{0x9e3779b97f4a7c15ULL * (i + 1), 0x632be59bd9b4e019ULL ^ i, 0, 0}};
        msg[i] = Scalar{{i * i + 1, i, 0, 0}};
        const Scalar* pk = (i % 2) ? PK2 : PK;
        pks[2 * i] = pk[0], pks[2 * i + 1] = pk[1];
    }
    std::vector<Scalar> R;
    const auto u = schnorr_sign_batch(keys.data(), n, r.data(), msg.data(), n, G, R, ok, e);
    if (!schnorr_verify_all(pks.data(), n, u.data(), R.data(), msg.data(), w.data(), n, G, &bad, e) || bad != 0) return 4;
    msg[17].l[0] ^= 1;
    if (schnorr_verify_all(pks.data(), n, u.data(), R.data(), msg.data(), w.data(), n, G, &bad, e) || bad != 0) return 5;
    try {
        Scalar off[2] = {G[0], G[1]};
        off[1].l[0] ^= 1;
        schnorr_verify_all(pks.data(), n, u.data(), R.data(), msg.data(), w.data(), n, off, nullptr, e);
        return 6;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_POINT) return 7;
    }
    std::puts("msm mirror ok (GPU)");
    return 0;
}
