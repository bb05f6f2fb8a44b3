// encrypt_batch_varlen / decrypt_batch_varlen of the C++ mirror (include/poseidon252_b200.hpp) against the C ABI.  Built
// and run by tests/test_crypt_varlen_bindings.py.  Without a GPU the default engine cannot be created (no CPU fallback);
// with one, messages of every length 1..40 in one call equal p252::encrypt per item, decrypt back with every ok set, and
// an empty message throws InvalidIOPattern.
#include <cstdio>
#include <cstring>

#include "poseidon252_b200.hpp"

int main() {
    using namespace p252;
    std::vector<std::vector<Scalar>> messages;
    std::vector<Scalar> uv, nonces;
    for (uint64_t len = 40; len >= 1; --len) {
        std::vector<Scalar> m;
        for (uint64_t j = 0; j < len; ++j) m.push_back(Scalar{{len * 100 + j, j, 0, 0}});
        messages.push_back(m);
        uv.push_back(Scalar{{len, 1, 0, 0}});
        uv.push_back(Scalar{{len, 2, 0, 0}});
        nonces.push_back(Scalar{{len, 3, 0, 0}});
    }
    int ndev = 0;
    p252_device_count(&ndev);
    if (ndev == 0) {
        try {
            encrypt_batch_varlen(messages, uv.data(), nonces.data());
            return 1;   // no CPU fallback
        } catch (const Error& e) {
            if (e.code != P252_ERR_NO_DEVICE) return 2;
        }
        std::puts("crypt varlen mirror ok (no GPU)");
        return 0;
    }
    Engine e(0);
    const auto ciphers = encrypt_batch_varlen(messages, uv.data(), nonces.data(), e);
    if (ciphers.size() != messages.size()) return 3;
    for (size_t i = 0; i < messages.size(); ++i) {
        const Scalar secret[2] = {uv[2 * i], uv[2 * i + 1]};
        const auto want = encrypt(messages[i], secret, nonces[i], e);
        if (ciphers[i].size() != want.size() || std::memcmp(ciphers[i].data(), want.data(), want.size() * sizeof(Scalar))) return 4;
    }
    std::vector<uint8_t> ok;
    const auto back = decrypt_batch_varlen(ciphers, uv.data(), nonces.data(), ok, e);
    for (size_t i = 0; i < messages.size(); ++i)
        if (!ok[i] || back[i].size() != messages[i].size() ||
            std::memcmp(back[i].data(), messages[i].data(), messages[i].size() * sizeof(Scalar)))
            return 5;
    messages[7].clear();
    try {
        encrypt_batch_varlen(messages, uv.data(), nonces.data(), e);
        return 6;
    } catch (const Error& err) {
        if (err.code != P252_ERR_INVALID_IO_PATTERN) return 7;
    }
    std::puts("crypt varlen mirror ok (GPU)");
    return 0;
}
