// poseidon252_b200.hpp -- header-only C++17 host mirror of the dusk_poseidon public surface
// (src/lib.rs:13-31) above the C ABI of poseidon252_b200.h.  The reference is compiled
// (Rust) code and no Rust toolchain exists in this image, so the compiled host side is C++; the Rust
// binding a maintainer would add is shown in INTEGRATION.md / bindings/rust/.
//
//   dusk_poseidon::Domain                    -> p252::Domain
//   dusk_poseidon::Hash{new,output_len,update,finalize,digest}   (src/hash.rs:92-195)  -> p252::Hash
//   dusk_poseidon::{encrypt, decrypt}        (src/encryption.rs:62-95) -> p252::encrypt / p252::decrypt
//   dusk_poseidon::Error                     (src/error.rs:11-32)      -> p252::Error (exception)
//   NEW batch entries: Hash::digest_batch, Hash::digest_batch_varlen, Hash::finalize_batch, hades::permute_batch,
//   encrypt_batch, decrypt_batch, encrypt_batch_varlen, decrypt_batch_varlen, dhke / dhke_batch, encrypt_batch_dhke,
//   decrypt_batch_dhke, fixed_base / fixed_base_batch, encrypt_batch_ephemeral, stealth_address /
//   stealth_address_batch, owns / stealth_owns_batch, schnorr_sign / schnorr_sign_batch, schnorr_verify /
//   schnorr_verify_batch, nullifier / nullifier_batch, schnorr_sign_double / schnorr_sign_double_batch,
//   schnorr_verify_double / schnorr_verify_double_batch, note_sign_double_batch, point_from_bytes /
//   points_from_bytes_batch, point_to_bytes / points_to_bytes_batch, value_commit / value_commit_batch,
//   note_create_batch, note_open / note_open_batch, wallet_scan_batch, elgamal_encrypt_batch, elgamal_decrypt_batch,
//   note_sender_encrypt_batch, note_sender_decrypt_batch, jubjub_msm, schnorr_verify_all,
//   schnorr_verify_double_all, merkle4_build, hash_to_scalar_batch, scalars_from_bytes_wide.
// Scalars are p252_fr == BlsScalar.0 (Montgomery limbs); every digest runs on the GPU (batch of 1 for the
// single-item calls).  No CPU fallback: Engine's constructor throws without an sm_90 device.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "poseidon252_b200.h"

namespace p252 {

using Scalar = p252_fr;

enum class Domain : int {   // src/hash.rs:21-36
    Merkle4 = P252_DOMAIN_MERKLE4,
    Merkle2 = P252_DOMAIN_MERKLE2,
    Encryption = P252_DOMAIN_ENCRYPTION,
    Other = P252_DOMAIN_OTHER,
};

// src/error.rs:11-32 -- `code` is the p252_status (positive = dusk_poseidon::Error variant)
struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& what) : std::runtime_error(what), code(c) {}
    bool is_io_pattern_violation() const { return code == P252_ERR_IO_PATTERN_VIOLATION; }
    bool is_decryption_failed() const { return code == P252_ERR_DECRYPTION_FAILED; }
};

inline void check(int rc, const p252_ctx* ctx = nullptr) {
    if (rc == P252_OK) return;
    std::string msg = p252_strerror(rc);
    if (ctx && *p252_last_error(ctx)) msg += std::string(" (") + p252_last_error(ctx) + ")";
    throw Error(rc, msg);
}

// u64::from(Domain), src/hash.rs:38-56
inline uint64_t domain_separator(Domain d) {
    uint64_t v = 0;
    check(p252_domain_separator(static_cast<int>(d), &v));
    return v;
}

class Engine {
public:
    explicit Engine(int device = 0, void* cuda_stream = nullptr) {
        check(cuda_stream ? p252_create_on_stream(device, cuda_stream, &ctx_) : p252_create(device, &ctx_));
    }
    ~Engine() { p252_destroy(ctx_); }
    Engine(const Engine&) = delete;
    Engine& operator=(const Engine&) = delete;
    p252_ctx* get() const { return ctx_; }
    void sync() { check(p252_sync(ctx_), ctx_); }
    uint64_t launch_count() const { return p252_launch_count(ctx_); }

    static Engine& default_engine() {
        static Engine e(0);
        return e;
    }

private:
    p252_ctx* ctx_ = nullptr;
};

namespace hades {
constexpr int WIDTH = P252_WIDTH;   // src/hades.rs:34

// n independent Safe::permute calls (src/hades/permutation/scalar.rs:25-27); states: n x 5, in place
inline void permute_batch(std::vector<Scalar>& states, Engine& e = Engine::default_engine()) {
    if (states.size() % WIDTH) throw Error(P252_ERR_INVALID_ARGUMENT, "states must hold n x 5 scalars");
    check(p252_permute_batch(e.get(), states.data(), states.size() / WIDTH, P252_MEM_HOST), e.get());
}
}  // namespace hades

class Hash {   // src/hash.rs:92-96
public:
    explicit Hash(Domain domain, Engine* e = nullptr) : domain_(domain), engine_(e) {}

    // src/hash.rs:111-115
    void output_len(size_t n) {
        if (domain_ == Domain::Other && n > 0) output_len_ = n;
    }
    // src/hash.rs:118-120 (the reference borrows the slice; this mirror borrows pointer + length)
    void update(const Scalar* input, size_t len) { chunks_.push_back({input, len}); }
    void update(const std::vector<Scalar>& input) { update(input.data(), input.size()); }

    // src/hash.rs:128-155.  Throws Error where the reference panics on an invalid io-pattern.
    std::vector<Scalar> finalize() const {
        // io_pattern, src/hash.rs:62-85: one Absorb per chunk + Squeeze(output_len)
        std::vector<uint32_t> calls;
        std::vector<Scalar> all;
        size_t total = 0;
        for (auto& c : chunks_) {
            calls.push_back(0x80000000u | static_cast<uint32_t>(c.len));
            all.insert(all.end(), c.ptr, c.ptr + c.len);
            total += c.len;
        }
        calls.push_back(static_cast<uint32_t>(output_len_));
        if ((domain_ == Domain::Merkle2 && (total != 2 || output_len_ != 1)) ||
            (domain_ == Domain::Merkle4 && (total != 4 || output_len_ != 1)))
            throw Error(P252_ERR_IO_PATTERN_VIOLATION, p252_strerror(P252_ERR_IO_PATTERN_VIOLATION));
        Scalar tag;
        check(p252_tag(calls.data(), calls.size(), domain_separator(domain_), &tag));
        std::vector<Scalar> out(output_len_);
        Engine& e = engine_ ? *engine_ : Engine::default_engine();
        check(p252_digest_batch(e.get(), &tag, all.data(), 1, total, out.data(), output_len_, P252_MEM_HOST), e.get());
        return out;
    }

    // src/hash.rs:191-195
    static std::vector<Scalar> digest(Domain domain, const std::vector<Scalar>& input, Engine* e = nullptr) {
        Hash h(domain, e);
        h.update(input);
        return h.finalize();
    }

    // NEW: n independent Hash::digest(domain, in[i*in_len .. (i+1)*in_len]) -> n x out_len
    static std::vector<Scalar> digest_batch(Domain domain, const Scalar* in, size_t n, size_t in_len,
                                            size_t output_len = 1, Engine* e = nullptr) {
        const size_t ol = (domain == Domain::Other && output_len > 0) ? output_len : 1;
        std::vector<Scalar> out(n * ol);
        Engine& eng = e ? *e : Engine::default_engine();
        check(p252_hash_batch(eng.get(), static_cast<int>(domain), in, n, in_len, out.data(), ol, P252_MEM_HOST),
              eng.get());
        return out;
    }

    // NEW: Hash::digest(domain, inputs[i]) for inputs of any lengths, one device call (p252_hash_batch_varlen);
    // output_len follows src/hash.rs:111-115.  Throws Error like Hash::finalize for an invalid item (nothing computed).
    static std::vector<std::vector<Scalar>> digest_batch_varlen(Domain domain, const std::vector<std::vector<Scalar>>& inputs,
                                                                size_t output_len = 1, Engine& e = Engine::default_engine()) {
        const size_t ol = (domain == Domain::Other && output_len > 0) ? output_len : 1;
        std::vector<Scalar> data;
        std::vector<uint64_t> offsets{0};
        size_t longest = 1;
        for (auto& in : inputs) {
            data.insert(data.end(), in.begin(), in.end());
            offsets.push_back(data.size());
            longest = in.size() > longest ? in.size() : longest;
        }
        std::vector<Scalar> out(inputs.size() * ol);
        check(p252_hash_batch_varlen(e.get(), static_cast<int>(domain), data.data(), data.size(), offsets.data(), inputs.size(),
                                     longest, out.data(), ol, nullptr, P252_MEM_HOST),
              e.get());
        std::vector<std::vector<Scalar>> res(inputs.size());
        for (size_t i = 0; i < res.size(); ++i) res[i].assign(out.begin() + i * ol, out.begin() + (i + 1) * ol);
        return res;
    }

    // NEW: hashes[i].finalize(), or hashes[i].finalize_truncated() where truncated[i] (empty: none truncated), for
    // hashes of any domains, update() chunks and output lengths, one device call (p252_hash_batch_mixed).  A truncated
    // item's rows are the raw limbs masked to 250 bits (JubJubScalar::from_raw's input).  Throws the Error
    // Hash::finalize throws for the lowest-index invalid hash before anything runs.
    static std::vector<std::vector<Scalar>> finalize_batch(const std::vector<Hash>& hashes,
                                                           const std::vector<bool>& truncated = {}, Engine* e = nullptr) {
        if (!truncated.empty() && truncated.size() != hashes.size())
            throw Error(P252_ERR_INVALID_ARGUMENT, "truncated must be empty or hold one flag per hash");
        std::vector<uint8_t> mode;
        std::vector<Scalar> data;
        std::vector<uint64_t> offsets{0}, out_offsets{0};
        size_t longest = 1, longest_out = 1;
        for (size_t i = 0; i < hashes.size(); ++i) {
            const Hash& h = hashes[i];
            size_t total = 0;
            bool empty_chunk = h.chunks_.empty();
            for (auto& c : h.chunks_) {
                data.insert(data.end(), c.ptr, c.ptr + c.len);
                total += c.len;
                empty_chunk = empty_chunk || c.len == 0;
            }
            if ((h.domain_ == Domain::Merkle2 && (total != 2 || h.output_len_ != 1)) ||
                (h.domain_ == Domain::Merkle4 && (total != 4 || h.output_len_ != 1)))
                throw Error(P252_ERR_IO_PATTERN_VIOLATION, p252_strerror(P252_ERR_IO_PATTERN_VIOLATION));
            if (empty_chunk) throw Error(P252_ERR_INVALID_IO_PATTERN, p252_strerror(P252_ERR_INVALID_IO_PATTERN));
            const bool trunc = !truncated.empty() && truncated[i];
            mode.push_back(static_cast<uint8_t>(static_cast<int>(h.domain_) | (trunc ? P252_MIXED_TRUNCATED : 0)));
            offsets.push_back(data.size());
            out_offsets.push_back(out_offsets.back() + h.output_len_);
            longest = std::max(longest, total);
            longest_out = std::max(longest_out, h.output_len_);
        }
        std::vector<Scalar> out(out_offsets.back());
        Engine& eng = e ? *e : Engine::default_engine();
        check(p252_hash_batch_mixed(eng.get(), mode.data(), data.data(), data.size(), offsets.data(), hashes.size(),
                                    longest, out.data(), out.size(), out_offsets.data(), longest_out, nullptr,
                                    P252_MEM_HOST),
              eng.get());
        std::vector<std::vector<Scalar>> res(hashes.size());
        for (size_t i = 0; i < res.size(); ++i)
            res[i].assign(out.begin() + out_offsets[i], out.begin() + out_offsets[i + 1]);
        return res;
    }

private:
    struct Chunk {
        const Scalar* ptr;
        size_t len;
    };
    Domain domain_;
    Engine* engine_;
    std::vector<Chunk> chunks_;
    size_t output_len_ = 1;
};

// NEW: BlsScalar::hash_to_scalar of byte strings of any lengths (empty ones included), one device call
// (p252_hash_to_scalar_batch): BLAKE2b-512, then from_bytes_wide, as Montgomery scalars ready to be a Schnorr msg.
// Throws Error(P252_ERR_INVALID_ARGUMENT) for a message longer than P252_HASH_TO_SCALAR_MAX_LEN (nothing computed).
inline std::vector<Scalar> hash_to_scalar_batch(const std::vector<std::vector<uint8_t>>& messages,
                                                Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> data;
    std::vector<uint64_t> offsets{0};
    size_t longest = 0;
    for (auto& m : messages) {
        data.insert(data.end(), m.begin(), m.end());
        offsets.push_back(data.size());
        longest = m.size() > longest ? m.size() : longest;
    }
    std::vector<Scalar> out(messages.size());
    check(p252_hash_to_scalar_batch(e.get(), data.data(), data.size(), offsets.data(), messages.size(), longest, out.data(),
                                    nullptr, P252_MEM_HOST),
          e.get());
    return out;
}
// NEW: BlsScalar::from_bytes_wide of n rows of 64 bytes (p252_scalars_from_bytes_wide); every row is valid
inline std::vector<Scalar> scalars_from_bytes_wide(const uint8_t* bytes, size_t n, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> out(n);
    check(p252_scalars_from_bytes_wide(e.get(), bytes, n, out.data(), P252_MEM_HOST), e.get());
    return out;
}

// src/encryption.rs:62-74; shared_secret = (u, v) of the JubJubAffine point (src/encryption.rs:71)
inline std::vector<Scalar> encrypt(const std::vector<Scalar>& message, const Scalar (&shared_secret_uv)[2],
                                   const Scalar& nonce, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> cipher(message.size() + 1);
    int rc = p252_encrypt_batch(e.get(), message.data(), 1, message.size(), shared_secret_uv, &nonce, cipher.data(),
                                P252_MEM_HOST);
    if (rc > 0) rc = P252_ERR_ENCRYPTION_FAILED;   // dusk-safe maps pattern errors of encrypt
    check(rc, e.get());
    return cipher;
}

// src/encryption.rs:83-95; throws Error{P252_ERR_DECRYPTION_FAILED} like Err(Error::DecryptionFailed)
inline std::vector<Scalar> decrypt(const std::vector<Scalar>& cipher, const Scalar (&shared_secret_uv)[2],
                                   const Scalar& nonce, Engine& e = Engine::default_engine()) {
    if (cipher.size() < 2) throw Error(P252_ERR_DECRYPTION_FAILED, p252_strerror(P252_ERR_DECRYPTION_FAILED));
    std::vector<Scalar> msg(cipher.size() - 1);
    uint8_t ok = 0;
    size_t failed = 0;
    check(p252_decrypt_batch(e.get(), cipher.data(), 1, msg.size(), shared_secret_uv, &nonce, msg.data(), &ok, &failed,
                             P252_MEM_HOST),
          e.get());
    if (!ok) throw Error(P252_ERR_DECRYPTION_FAILED, p252_strerror(P252_ERR_DECRYPTION_FAILED));
    return msg;
}

// NEW batch forms (item-major): msg n x L, secrets n x 2, nonces n  ->  cipher n x (L+1)
inline std::vector<Scalar> encrypt_batch(const Scalar* msg, size_t n, size_t L, const Scalar* secrets_uv,
                                         const Scalar* nonces, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> cipher(n * (L + 1));
    check(p252_encrypt_batch(e.get(), msg, n, L, secrets_uv, nonces, cipher.data(), P252_MEM_HOST), e.get());
    return cipher;
}
// returns the messages; ok[i] == 0 marks items for which the reference returns DecryptionFailed
inline std::vector<Scalar> decrypt_batch(const Scalar* cipher, size_t n, size_t L, const Scalar* secrets_uv,
                                         const Scalar* nonces, std::vector<uint8_t>& ok,
                                         Engine& e = Engine::default_engine()) {
    std::vector<Scalar> msg(n * L);
    ok.assign(n, 0);
    check(p252_decrypt_batch(e.get(), cipher, n, L, secrets_uv, nonces, msg.data(), ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return msg;
}

// NEW: encrypt / decrypt of messages of any lengths in one device call (p252_encrypt_batch_varlen /
// p252_decrypt_batch_varlen); secrets n x 2, nonces n.  Throws Error for an invalid item (nothing computed).
namespace detail {
inline size_t pack(const std::vector<std::vector<Scalar>>& items, std::vector<Scalar>& data, std::vector<uint64_t>& offsets) {
    size_t longest = 0;
    offsets.assign(1, 0);
    for (auto& it : items) {
        data.insert(data.end(), it.begin(), it.end());
        offsets.push_back(data.size());
        longest = it.size() > longest ? it.size() : longest;
    }
    return longest;
}
}  // namespace detail

inline std::vector<std::vector<Scalar>> encrypt_batch_varlen(const std::vector<std::vector<Scalar>>& messages,
                                                             const Scalar* secrets_uv, const Scalar* nonces,
                                                             Engine& e = Engine::default_engine()) {
    std::vector<Scalar> data;
    std::vector<uint64_t> off;
    const size_t longest = detail::pack(messages, data, off);
    const size_t n = messages.size();
    std::vector<Scalar> cipher(data.size() + n);
    check(p252_encrypt_batch_varlen(e.get(), data.data(), data.size(), off.data(), n, longest ? longest : 1, secrets_uv, nonces,
                                    cipher.data(), nullptr, P252_MEM_HOST),
          e.get());
    std::vector<std::vector<Scalar>> res(n);
    for (size_t i = 0; i < n; ++i) res[i].assign(cipher.begin() + off[i] + i, cipher.begin() + off[i + 1] + i + 1);
    return res;
}
// returns the messages; ok[i] == 0 marks items for which the reference returns DecryptionFailed (their message is zero)
inline std::vector<std::vector<Scalar>> decrypt_batch_varlen(const std::vector<std::vector<Scalar>>& ciphers,
                                                             const Scalar* secrets_uv, const Scalar* nonces,
                                                             std::vector<uint8_t>& ok, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> data;
    std::vector<uint64_t> off;
    const size_t longest = detail::pack(ciphers, data, off);
    const size_t n = ciphers.size();
    std::vector<Scalar> msg(data.size() > n ? data.size() - n : 0);
    ok.assign(n, 0);
    check(p252_decrypt_batch_varlen(e.get(), data.data(), data.size(), off.data(), n, longest > 1 ? longest - 1 : 1, secrets_uv,
                                    nonces, msg.data(), ok.data(), nullptr, nullptr, P252_MEM_HOST),
          e.get());
    std::vector<std::vector<Scalar>> res(n);
    for (size_t i = 0; i < n; ++i) res[i].assign(msg.begin() + (off[i] - i), msg.begin() + (off[i + 1] - i - 1));
    return res;
}

// NEW: JubJub key exchange (p252_dhke_batch) and encrypt / decrypt with the shared secret derived on the device
// (p252_{en,de}crypt_batch_dhke).  Secrets are canonical p252_jscalar (JubJubScalar::to_bytes), points (u, v) pairs;
// n_secret and n_public are each 1 (broadcast) or n.  ok[i] == 0 marks an invalid item (secret >= r_J or a point off the
// curve; for decrypt also an authentication failure) with a zeroed output row.
using JubJubScalar = p252_jscalar;
// returns n x 2 scalars: (u, v) of [secret] public per item
inline std::vector<Scalar> dhke_batch(const JubJubScalar* secrets, size_t n_secret, const Scalar* publics_uv, size_t n_public,
                                      size_t n, std::vector<uint8_t>& ok, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> shared(2 * n);
    ok.assign(n, 0);
    check(p252_dhke_batch(e.get(), secrets, n_secret, publics_uv, n_public, n, shared.data(), ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return shared;
}
// dhke(secret, public) for one item; throws Error(P252_ERR_INVALID_POINT) like the reference's Error::InvalidPoint
inline void dhke(const JubJubScalar& secret, const Scalar (&public_uv)[2], Scalar (&shared_uv)[2],
                 Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto r = dhke_batch(&secret, 1, public_uv, 1, 1, ok, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    shared_uv[0] = r[0];
    shared_uv[1] = r[1];
}
// msg n x L -> cipher n x (L+1)
inline std::vector<Scalar> encrypt_batch_dhke(const Scalar* msg, size_t n, size_t L, const JubJubScalar* secrets, size_t n_secret,
                                              const Scalar* publics_uv, size_t n_public, const Scalar* nonces,
                                              std::vector<uint8_t>& ok, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> cipher(n * (L + 1));
    ok.assign(n, 0);
    check(p252_encrypt_batch_dhke(e.get(), msg, n, L, secrets, n_secret, publics_uv, n_public, nonces, cipher.data(), ok.data(),
                                  nullptr, P252_MEM_HOST),
          e.get());
    return cipher;
}
// cipher n x (L+1) -> msg n x L
inline std::vector<Scalar> decrypt_batch_dhke(const Scalar* cipher, size_t n, size_t L, const JubJubScalar* secrets,
                                              size_t n_secret, const Scalar* publics_uv, size_t n_public, const Scalar* nonces,
                                              std::vector<uint8_t>& ok, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> msg(n * L);
    ok.assign(n, 0);
    check(p252_decrypt_batch_dhke(e.get(), cipher, n, L, secrets, n_secret, publics_uv, n_public, nonces, msg.data(), ok.data(),
                                  nullptr, P252_MEM_HOST),
          e.get());
    return msg;
}

// NEW: fixed-base scalar multiplication (p252_fixed_base_batch) and the sender's encrypt batch
// (p252_encrypt_batch_ephemeral).  base_uv is the caller's base point (u, v), e.g. dusk_jubjub::GENERATOR's; there is no
// built-in generator.  A base off the curve throws Error(P252_ERR_INVALID_POINT); ok[i] == 0 marks an invalid item (secret
// >= r_J, or in the fused call a public key off the curve) with zeroed output rows.
// returns n x 2 scalars: (u, v) of [secrets[i]] base
inline std::vector<Scalar> fixed_base_batch(const JubJubScalar* secrets, size_t n, const Scalar (&base_uv)[2],
                                            std::vector<uint8_t>& ok, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> out(2 * n);
    ok.assign(n, 0);
    check(p252_fixed_base_batch(e.get(), base_uv, secrets, n, out.data(), ok.data(), nullptr, P252_MEM_HOST), e.get());
    return out;
}
// [secret] base for one item, e.g. a public key; throws Error(P252_ERR_INVALID_POINT) for a secret >= r_J
inline void fixed_base(const JubJubScalar& secret, const Scalar (&base_uv)[2], Scalar (&out_uv)[2],
                       Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto r = fixed_base_batch(&secret, 1, base_uv, ok, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    out_uv[0] = r[0];
    out_uv[1] = r[1];
}
// msg n x L -> cipher n x (L+1); R receives n x 2 scalars, the ephemeral keys [r_i] base
inline std::vector<Scalar> encrypt_batch_ephemeral(const Scalar* msg, size_t n, size_t L, const JubJubScalar* r,
                                                   const Scalar (&base_uv)[2], const Scalar* publics_uv, size_t n_public,
                                                   const Scalar* nonces, std::vector<Scalar>& R, std::vector<uint8_t>& ok,
                                                   Engine& e = Engine::default_engine()) {
    std::vector<Scalar> cipher(n * (L + 1));
    R.assign(2 * n, Scalar{});
    ok.assign(n, 0);
    check(p252_encrypt_batch_ephemeral(e.get(), msg, n, L, r, base_uv, publics_uv, n_public, nonces, cipher.data(), R.data(),
                                       ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return cipher;
}

// NEW: stealth addresses (p252_stealth_address_batch / p252_stealth_owns_batch).  The sender makes R = [r] G and
// note_pk = [hash([r] A)] G + B for the receiver's key (A, B); the receiver with view key a and spend key B owns a note iff
// note_pk == [hash([a] R)] G + B.  base_uv is the caller's G (no built-in generator); a G or receiver B off the curve
// throws Error(P252_ERR_INVALID_POINT).  publics_A / publics_B hold 1 or n points each (n_public).
// returns n x 2 scalars, the note keys; R receives n x 2 scalars; ok[i] == 0 marks an invalid item (zeroed rows)
inline std::vector<Scalar> stealth_address_batch(const JubJubScalar* r, size_t n, const Scalar (&base_uv)[2],
                                                 const Scalar* publics_A, const Scalar* publics_B, size_t n_public,
                                                 std::vector<Scalar>& R, std::vector<uint8_t>& ok,
                                                 Engine& e = Engine::default_engine()) {
    std::vector<Scalar> note_pk(2 * n);
    R.assign(2 * n, Scalar{});
    ok.assign(n, 0);
    check(p252_stealth_address_batch(e.get(), r, n, base_uv, publics_A, publics_B, n_public, R.data(), note_pk.data(),
                                     ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return note_pk;
}
// one note; throws Error(P252_ERR_INVALID_POINT) for r >= r_J or a receiver key off the curve
inline void stealth_address(const JubJubScalar& r, const Scalar (&base_uv)[2], const Scalar (&A_uv)[2], const Scalar (&B_uv)[2],
                            Scalar (&R_uv)[2], Scalar (&note_pk_uv)[2], Engine& e = Engine::default_engine()) {
    std::vector<Scalar> R;
    std::vector<uint8_t> ok;
    const auto pk = stealth_address_batch(&r, 1, base_uv, A_uv, B_uv, 1, R, ok, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    R_uv[0] = R[0], R_uv[1] = R[1];
    note_pk_uv[0] = pk[0], note_pk_uv[1] = pk[1];
}
// R and note_pk n x 2 scalars each; returns owned[i] (0 also for an invalid item); n_owned / n_invalid may be null
inline std::vector<uint8_t> stealth_owns_batch(const JubJubScalar& view_a, const Scalar (&spend_B_uv)[2],
                                               const Scalar (&base_uv)[2], const Scalar* R, const Scalar* note_pk, size_t n,
                                               size_t* n_owned = nullptr, size_t* n_invalid = nullptr,
                                               Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> owned(n, 0);
    check(p252_stealth_owns_batch(e.get(), &view_a, spend_B_uv, base_uv, R, note_pk, n, owned.data(), n_owned, n_invalid,
                                  P252_MEM_HOST),
          e.get());
    return owned;
}
// ViewKey::owns for one note; throws Error(P252_ERR_INVALID_POINT) for a view key >= r_J, an R off the curve or a
// note_pk coordinate >= p
inline bool owns(const JubJubScalar& view_a, const Scalar (&spend_B_uv)[2], const Scalar (&base_uv)[2], const Scalar (&R_uv)[2],
                 const Scalar (&note_pk_uv)[2], Engine& e = Engine::default_engine()) {
    size_t invalid = 0;
    const auto owned = stealth_owns_batch(view_a, spend_B_uv, base_uv, R_uv, note_pk_uv, 1, nullptr, &invalid, e);
    if (invalid) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    return owned[0] != 0;
}

// NEW: Schnorr signatures over JubJub (p252_schnorr_sign_batch / p252_schnorr_verify_batch), jubjub-schnorr's
// SecretKey::sign / PublicKey::verify: R = [r] G, u = (r - c sk) mod r_J with c = challenge(R, m) =
// Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0]; verified iff [u] G + [c] PK == R.  base_uv is the caller's G;
// a G off the curve throws Error(P252_ERR_INVALID_POINT).  r is one fresh secret nonce per message (never reused).
// sk holds 1 or n keys (n_secret); returns the n scalars u; R receives n x 2 scalars; ok[i] == 0 marks an invalid item
inline std::vector<JubJubScalar> schnorr_sign_batch(const JubJubScalar* sk, size_t n_secret, const JubJubScalar* r,
                                                    const Scalar* msg, size_t n, const Scalar (&base_uv)[2],
                                                    std::vector<Scalar>& R, std::vector<uint8_t>& ok,
                                                    Engine& e = Engine::default_engine()) {
    std::vector<JubJubScalar> u(n);
    R.assign(2 * n, Scalar{});
    ok.assign(n, 0);
    check(p252_schnorr_sign_batch(e.get(), sk, n_secret, r, msg, n, base_uv, u.data(), R.data(), ok.data(), nullptr,
                                  P252_MEM_HOST),
          e.get());
    return u;
}
// one signature (u, R); throws Error(P252_ERR_INVALID_POINT) for sk or r >= r_J or msg >= p
inline void schnorr_sign(const JubJubScalar& sk, const JubJubScalar& r, const Scalar& msg, const Scalar (&base_uv)[2],
                         JubJubScalar& u, Scalar (&R_uv)[2], Engine& e = Engine::default_engine()) {
    std::vector<Scalar> R;
    std::vector<uint8_t> ok;
    const auto us = schnorr_sign_batch(&sk, 1, &r, &msg, 1, base_uv, R, ok, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    u = us[0];
    R_uv[0] = R[0], R_uv[1] = R[1];
}
// pk holds 1 or n points (n_public), R n x 2 scalars; returns verified[i] (0 also for an invalid item); n_verified /
// n_invalid may be null
inline std::vector<uint8_t> schnorr_verify_batch(const Scalar* pk, size_t n_public, const JubJubScalar* u, const Scalar* R,
                                                 const Scalar* msg, size_t n, const Scalar (&base_uv)[2],
                                                 size_t* n_verified = nullptr, size_t* n_invalid = nullptr,
                                                 Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> verified(n, 0);
    check(p252_schnorr_verify_batch(e.get(), pk, n_public, u, R, msg, n, base_uv, verified.data(), n_verified, n_invalid,
                                    P252_MEM_HOST),
          e.get());
    return verified;
}
// PublicKey::verify for one signature; throws Error(P252_ERR_INVALID_POINT) for u >= r_J, msg >= p, an R coordinate
// >= p or a key off the curve
inline bool schnorr_verify(const Scalar (&pk_uv)[2], const JubJubScalar& u, const Scalar (&R_uv)[2], const Scalar& msg,
                           const Scalar (&base_uv)[2], Engine& e = Engine::default_engine()) {
    size_t invalid = 0;
    const auto verified = schnorr_verify_batch(pk_uv, 1, &u, R_uv, &msg, 1, base_uv, nullptr, &invalid, e);
    if (invalid) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    return verified[0] != 0;
}

// NEW: Phoenix note nullifiers (p252_nullifier_batch): nullifier = Hash::digest(Domain::Other, [pk'.u, pk'.v, pos])[0] with
// pk' = [note_sk] G' and note_sk = (hash([a] R) + b) mod r_J, hash the stealth calls' truncated digest.  base_uv is the
// caller's G' (no built-in generator); a G' off the curve throws Error(P252_ERR_INVALID_POINT).  a and b hold 1 or n keys
// each (n_secret); R holds n x 2 scalars and pos n positions.  Returns the n nullifiers; ok[i] == 0 marks an invalid item
// (a or b >= r_J, R off the curve), whose nullifier is zeroed.  n_invalid may be null.
inline std::vector<Scalar> nullifier_batch(const JubJubScalar* a, const JubJubScalar* b, size_t n_secret,
                                           const Scalar (&base_uv)[2], const Scalar* R, const uint64_t* pos, size_t n,
                                           std::vector<uint8_t>& ok, size_t* n_invalid = nullptr,
                                           Engine& e = Engine::default_engine()) {
    std::vector<Scalar> out(n);
    ok.assign(n, 0);
    check(p252_nullifier_batch(e.get(), a, b, n_secret, base_uv, R, pos, n, out.data(), ok.data(), n_invalid, P252_MEM_HOST),
          e.get());
    return out;
}
// Note::gen_nullifier for one note; throws Error(P252_ERR_INVALID_POINT) for a or b >= r_J or an R off the curve
inline Scalar nullifier(const JubJubScalar& a, const JubJubScalar& b, const Scalar (&base_uv)[2], const Scalar (&R_uv)[2],
                        uint64_t pos, Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto r = nullifier_batch(&a, &b, 1, base_uv, R_uv, &pos, 1, ok, nullptr, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    return r[0];
}

// NEW: double-key Schnorr signatures over G and G' (p252_schnorr_sign_double_batch / p252_schnorr_verify_double_batch),
// jubjub-schnorr's SecretKey::sign_double / SignatureDouble::verify: R = [r] G, R' = [r] G', u = (r - c sk) mod r_J with
// c = challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0]; verified iff
// [u] G + [c] PK == R and [u] G' + [c] PK' == R'.  G_uv and Gp_uv are the caller's G and G' (no built-in generator);
// either off the curve throws Error(P252_ERR_INVALID_POINT).  r is one fresh secret nonce per message (never reused).
// sk holds 1 or n keys (n_secret); returns the n scalars u; R and Rp receive n x 2 scalars each; ok[i] == 0 marks an
// invalid item, whose rows are zeroed
inline std::vector<JubJubScalar> schnorr_sign_double_batch(const JubJubScalar* sk, size_t n_secret, const JubJubScalar* r,
                                                           const Scalar* msg, size_t n, const Scalar (&G_uv)[2],
                                                           const Scalar (&Gp_uv)[2], std::vector<Scalar>& R,
                                                           std::vector<Scalar>& Rp, std::vector<uint8_t>& ok,
                                                           Engine& e = Engine::default_engine()) {
    std::vector<JubJubScalar> u(n);
    R.assign(2 * n, Scalar{});
    Rp.assign(2 * n, Scalar{});
    ok.assign(n, 0);
    check(p252_schnorr_sign_double_batch(e.get(), sk, n_secret, r, msg, n, G_uv, Gp_uv, u.data(), R.data(), Rp.data(),
                                         ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return u;
}
// one double-key signature (u, R, R'); throws Error(P252_ERR_INVALID_POINT) for sk or r >= r_J or msg >= p
inline void schnorr_sign_double(const JubJubScalar& sk, const JubJubScalar& r, const Scalar& msg, const Scalar (&G_uv)[2],
                                const Scalar (&Gp_uv)[2], JubJubScalar& u, Scalar (&R_uv)[2], Scalar (&Rp_uv)[2],
                                Engine& e = Engine::default_engine()) {
    std::vector<Scalar> R, Rp;
    std::vector<uint8_t> ok;
    const auto us = schnorr_sign_double_batch(&sk, 1, &r, &msg, 1, G_uv, Gp_uv, R, Rp, ok, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    u = us[0];
    R_uv[0] = R[0], R_uv[1] = R[1], Rp_uv[0] = Rp[0], Rp_uv[1] = Rp[1];
}
// pk and pkp hold 1 or n points each (n_public), R and Rp n x 2 scalars; returns verified[i] (0 also for an invalid
// item); n_verified / n_invalid may be null
inline std::vector<uint8_t> schnorr_verify_double_batch(const Scalar* pk, const Scalar* pkp, size_t n_public,
                                                        const JubJubScalar* u, const Scalar* R, const Scalar* Rp,
                                                        const Scalar* msg, size_t n, const Scalar (&G_uv)[2],
                                                        const Scalar (&Gp_uv)[2], size_t* n_verified = nullptr,
                                                        size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> verified(n, 0);
    check(p252_schnorr_verify_double_batch(e.get(), pk, pkp, n_public, u, R, Rp, msg, n, G_uv, Gp_uv, verified.data(),
                                           n_verified, n_invalid, P252_MEM_HOST),
          e.get());
    return verified;
}
// SignatureDouble::verify for one signature; throws Error(P252_ERR_INVALID_POINT) for u >= r_J, msg >= p, a coordinate
// of R or R' >= p or a key off the curve
inline bool schnorr_verify_double(const Scalar (&pk_uv)[2], const Scalar (&pkp_uv)[2], const JubJubScalar& u,
                                  const Scalar (&R_uv)[2], const Scalar (&Rp_uv)[2], const Scalar& msg,
                                  const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2], Engine& e = Engine::default_engine()) {
    size_t invalid = 0;
    const auto verified = schnorr_verify_double_batch(pk_uv, pkp_uv, 1, &u, R_uv, Rp_uv, &msg, 1, G_uv, Gp_uv, nullptr,
                                                      &invalid, e);
    if (invalid) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    return verified[0] != 0;
}
// NEW: spending notes (p252_note_sign_double_batch): the double-key signature of msg[i] under the note secret key
// note_sk = (hash([a] note_R[i]) + b) mod r_J, whose key pair is (note_pk, pk') = ([note_sk] G, [note_sk] G').  a and b
// hold 1 or n keys each (n_secret); note_R holds n x 2 scalars.  Returns the n scalars u; R, Rp and pkp (pk', the spend
// proof's witness: it links the spend to the note, keep it private) receive n x 2 scalars each; ok[i] == 0 marks an
// invalid item (a, b or r >= r_J, note_R off the curve, msg >= p), whose rows are zeroed.  n_invalid may be null.
inline std::vector<JubJubScalar> note_sign_double_batch(const JubJubScalar* a, const JubJubScalar* b, size_t n_secret,
                                                        const Scalar* note_R, const JubJubScalar* r, const Scalar* msg,
                                                        size_t n, const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2],
                                                        std::vector<Scalar>& R, std::vector<Scalar>& Rp,
                                                        std::vector<Scalar>& pkp, std::vector<uint8_t>& ok,
                                                        size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    std::vector<JubJubScalar> u(n);
    R.assign(2 * n, Scalar{});
    Rp.assign(2 * n, Scalar{});
    pkp.assign(2 * n, Scalar{});
    ok.assign(n, 0);
    check(p252_note_sign_double_batch(e.get(), a, b, n_secret, note_R, r, msg, n, G_uv, Gp_uv, u.data(), R.data(), Rp.data(),
                                      pkp.data(), ok.data(), n_invalid, P252_MEM_HOST),
          e.get());
    return u;
}

// NEW: JubJub point compression (p252_points_from_bytes / p252_points_to_bytes), dusk-jubjub's JubJubAffine::from_bytes /
// to_bytes: the 32 little-endian bytes of canonical v with the low bit of canonical u in bit 255.
// bytes holds n x 32 bytes; returns n x 2 scalars (u, v); ok[i] == 0 marks an encoding with v >= p or u^2 not a square,
// whose row is (0, 0).  n_invalid may be null.
inline std::vector<Scalar> points_from_bytes_batch(const uint8_t* bytes, size_t n, std::vector<uint8_t>& ok,
                                                   size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> uv(2 * n);
    ok.assign(n, 0);
    check(p252_points_from_bytes(e.get(), bytes, n, uv.data(), ok.data(), n_invalid, P252_MEM_HOST), e.get());
    return uv;
}
// uv holds n x 2 scalars; returns n x 32 bytes; ok[i] == 0 marks a coordinate >= p or a point off the curve, whose
// encoding is 32 bytes of 0xff.  n_invalid may be null.
inline std::vector<uint8_t> points_to_bytes_batch(const Scalar* uv, size_t n, std::vector<uint8_t>& ok,
                                                  size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> bytes(32 * n);
    ok.assign(n, 0);
    check(p252_points_to_bytes(e.get(), uv, n, bytes.data(), ok.data(), n_invalid, P252_MEM_HOST), e.get());
    return bytes;
}
// JubJubAffine::from_bytes for one encoding; throws Error(P252_ERR_INVALID_POINT) for an invalid one
inline void point_from_bytes(const uint8_t (&bytes)[32], Scalar (&uv)[2], Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto r = points_from_bytes_batch(bytes, 1, ok, nullptr, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    uv[0] = r[0], uv[1] = r[1];
}
// JubJubAffine::to_bytes for one point; throws Error(P252_ERR_INVALID_POINT) for a coordinate >= p or a point off the curve
inline void point_to_bytes(const Scalar (&uv)[2], uint8_t (&bytes)[32], Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto r = points_to_bytes_batch(uv, 1, ok, nullptr, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    std::copy(r.begin(), r.end(), bytes);
}

// NEW: Phoenix note values (p252_value_commit_batch / p252_note_create_batch / p252_note_open_batch): the value commitment
// C = [v] G + [blinder] G' (v a u64, blinder < r_J), obfuscated notes for the receiver (A, B) -- R = [r] G, S = [r] A,
// note_pk = [hash(S)] G + B, C, cipher = encrypt([Fr(v), Fr(blinder)], S, nonce) (3 scalars) -- and the wallet's checked
// opening: (m0, m1) = decrypt(cipher, [a] R, nonce) opens the note iff the authentication passes, m0 < 2^64, m1 < r_J and
// [m0] G + [m1] G' == C.  G_uv and Gp_uv are the caller's G and G' (GENERATOR_NUMS); either off the curve throws
// Error(P252_ERR_INVALID_POINT).  ok[i] == 0 marks an invalid item (or a note that did not open), whose rows are zeroed.
// Returns the n commitments (2 scalars each)
inline std::vector<Scalar> value_commit_batch(const uint64_t* value, const JubJubScalar* blinder, size_t n,
                                              const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2], std::vector<uint8_t>& ok,
                                              size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    std::vector<Scalar> C(2 * n);
    ok.assign(n, 0);
    check(p252_value_commit_batch(e.get(), value, blinder, n, G_uv, Gp_uv, C.data(), ok.data(), n_invalid, P252_MEM_HOST),
          e.get());
    return C;
}
// one commitment; throws Error(P252_ERR_INVALID_POINT) for blinder >= r_J
inline void value_commit(uint64_t value, const JubJubScalar& blinder, const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2],
                         Scalar (&C_uv)[2], Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok;
    const auto C = value_commit_batch(&value, &blinder, 1, G_uv, Gp_uv, ok, nullptr, e);
    if (!ok[0]) throw Error(P252_ERR_INVALID_POINT, p252_strerror(P252_ERR_INVALID_POINT));
    C_uv[0] = C[0], C_uv[1] = C[1];
}
// A and B hold 1 or n points each (n_public); R, note_pk and C receive n x 2 scalars, cipher n x 3.  Returns ok
inline std::vector<uint8_t> note_create_batch(const JubJubScalar* r, const uint64_t* value, const JubJubScalar* blinder,
                                              const Scalar* nonce, size_t n, const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2],
                                              const Scalar* A, const Scalar* B, size_t n_public, std::vector<Scalar>& R,
                                              std::vector<Scalar>& note_pk, std::vector<Scalar>& C,
                                              std::vector<Scalar>& cipher, size_t* n_invalid = nullptr,
                                              Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok(n, 0);
    R.assign(2 * n, Scalar{});
    note_pk.assign(2 * n, Scalar{});
    C.assign(2 * n, Scalar{});
    cipher.assign(3 * n, Scalar{});
    check(p252_note_create_batch(e.get(), r, value, blinder, nonce, n, G_uv, Gp_uv, A, B, n_public, R.data(), note_pk.data(),
                                 C.data(), cipher.data(), ok.data(), n_invalid, P252_MEM_HOST),
          e.get());
    return ok;
}
// a holds 1 or n view keys (n_secret); R, C n x 2 scalars, cipher n x 3.  Returns the n values; blinder receives n
// scalars; n_failed (may be null) counts the items with ok == 0.  value and blinder are the spend proof's witnesses
inline std::vector<uint64_t> note_open_batch(const JubJubScalar* a, size_t n_secret, const Scalar* R, const Scalar* nonce,
                                             const Scalar* cipher, const Scalar* C, size_t n, const Scalar (&G_uv)[2],
                                             const Scalar (&Gp_uv)[2], std::vector<JubJubScalar>& blinder,
                                             std::vector<uint8_t>& ok, size_t* n_failed = nullptr,
                                             Engine& e = Engine::default_engine()) {
    std::vector<uint64_t> value(n, 0);
    blinder.assign(n, JubJubScalar{});
    ok.assign(n, 0);
    check(p252_note_open_batch(e.get(), a, n_secret, R, nonce, cipher, C, n, G_uv, Gp_uv, value.data(), blinder.data(),
                               ok.data(), n_failed, P252_MEM_HOST),
          e.get());
    return value;
}
// the opening of one note -> v; throws Error(P252_ERR_INVALID_POINT) for a >= r_J or an R off the curve, and
// Error(P252_ERR_DECRYPTION_FAILED) for a note that does not open
inline uint64_t note_open(const JubJubScalar& a, const Scalar (&R_uv)[2], const Scalar& nonce, const Scalar (&cipher)[3],
                          const Scalar (&C_uv)[2], const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2], JubJubScalar& blinder,
                          Engine& e = Engine::default_engine()) {
    std::vector<JubJubScalar> b;
    std::vector<uint8_t> ok;
    const auto v = note_open_batch(&a, 1, R_uv, &nonce, cipher, C_uv, 1, G_uv, Gp_uv, b, ok, nullptr, e);
    if (!ok[0]) {
        static const uint64_t order[4] = {0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL,
                                          0x0e7db4ea6533afa9ULL};   // r_J
        bool below = false;
        for (int k = 3; k >= 0; --k)
            if (a.l[k] != order[k]) {
                below = a.l[k] < order[k];
                break;
            }
        std::vector<uint8_t> on_curve;
        points_to_bytes_batch(R_uv, 1, on_curve, nullptr, e);
        const int code = below && on_curve[0] ? P252_ERR_DECRYPTION_FAILED : P252_ERR_INVALID_POINT;
        throw Error(code, p252_strerror(code));
    }
    blinder = b[0];
    return v[0];
}

// NEW: multi-key wallet scans (p252_wallet_scan_batch): for each note the smallest key j whose (a_j, B_j = [b_j] G) owns
// it (owner -1: none), and for owned notes the nullifier and the checked opening under that key; key_totals row j =
// {value_lo, value_hi, n_owned, n_opened}.  a, b: n_keys keys (1..P252_WALLET_MAX_KEYS); R, note_pk, C: n x 2 scalars;
// cipher n x 3.  G_uv / Gp_uv off the curve throw Error(P252_ERR_INVALID_POINT).  Returns every result and both counts.
struct WalletScan {
    std::vector<int32_t> owner;
    std::vector<Scalar> nullifier;
    std::vector<uint64_t> value;
    std::vector<JubJubScalar> blinder;
    std::vector<uint8_t> opened;
    std::vector<uint64_t> key_totals;   // n_keys x 4
    size_t n_invalid = 0, n_bad_keys = 0;
};
inline WalletScan wallet_scan_batch(const JubJubScalar* a, const JubJubScalar* b, size_t n_keys, const Scalar* R,
                                    const Scalar* note_pk, const uint64_t* pos, const Scalar* nonce, const Scalar* cipher,
                                    const Scalar* C, size_t n, const Scalar (&G_uv)[2], const Scalar (&Gp_uv)[2],
                                    Engine& e = Engine::default_engine()) {
    WalletScan w;
    w.owner.assign(n, -1);
    w.nullifier.assign(n, Scalar{});
    w.value.assign(n, 0);
    w.blinder.assign(n, JubJubScalar{});
    w.opened.assign(n, 0);
    w.key_totals.assign(4 * n_keys, 0);
    check(p252_wallet_scan_batch(e.get(), a, b, n_keys, R, note_pk, pos, nonce, cipher, C, n, G_uv, Gp_uv, w.owner.data(),
                                 w.nullifier.data(), w.value.data(), w.blinder.data(), w.opened.data(), w.key_totals.data(),
                                 &w.n_invalid, &w.n_bad_keys, P252_MEM_HOST),
          e.get());
    return w;
}

// NEW: JubJub ElGamal and the encrypted sender of a Phoenix note (p252_elgamal_encrypt_batch / p252_elgamal_decrypt_batch /
// p252_note_sender_encrypt_batch / p252_note_sender_decrypt_batch): (c1, c2) = ([r] G, M + [r] PK), M = c2 - [sk] c1
// (NOT authenticated: a wrong key gives another point); the sender field is [(c1_A, c2_A), (c1_B, c2_B)] under note_pk,
// opened with note_sk = (hash([a] R) + b) mod r_J only where [note_sk] G == note_pk.  Points are n x 2 scalars; pk, A and
// B hold 1 or n points (n_public / n_sender), sk, a and b 1 or n keys (n_secret); r one per message and blinder two per
// note [r_A, r_B], never reused.  G_uv off the curve throws Error(P252_ERR_INVALID_POINT).  ok[i] == 0 marks an item
// with zeroed rows (invalid; for the sender decrypt also not owned); the counts may be null.
inline std::vector<uint8_t> elgamal_encrypt_batch(const Scalar* pk, size_t n_public, const Scalar* msg, const JubJubScalar* r,
                                                  size_t n, const Scalar (&G_uv)[2], std::vector<Scalar>& c1,
                                                  std::vector<Scalar>& c2, size_t* n_invalid = nullptr,
                                                  Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok(n, 0);
    c1.assign(2 * n, Scalar{});
    c2.assign(2 * n, Scalar{});
    check(p252_elgamal_encrypt_batch(e.get(), pk, n_public, msg, r, n, G_uv, c1.data(), c2.data(), ok.data(), n_invalid,
                                     P252_MEM_HOST),
          e.get());
    return ok;
}
inline std::vector<Scalar> elgamal_decrypt_batch(const JubJubScalar* sk, size_t n_secret, const Scalar* c1, const Scalar* c2,
                                                 size_t n, std::vector<uint8_t>& ok, size_t* n_invalid = nullptr,
                                                 Engine& e = Engine::default_engine()) {
    std::vector<Scalar> msg(2 * n);
    ok.assign(n, 0);
    check(p252_elgamal_decrypt_batch(e.get(), sk, n_secret, c1, c2, n, msg.data(), ok.data(), n_invalid, P252_MEM_HOST),
          e.get());
    return msg;
}
// enc receives 8 scalars per note: [c1_A, c2_A, c1_B, c2_B]
inline std::vector<uint8_t> note_sender_encrypt_batch(const Scalar* note_pk, const Scalar* A, const Scalar* B, size_t n_sender,
                                                      const JubJubScalar* blinder, size_t n, const Scalar (&G_uv)[2],
                                                      std::vector<Scalar>& enc, size_t* n_invalid = nullptr,
                                                      Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok(n, 0);
    enc.assign(8 * n, Scalar{});
    check(p252_note_sender_encrypt_batch(e.get(), note_pk, A, B, n_sender, blinder, n, G_uv, enc.data(), ok.data(),
                                         n_invalid, P252_MEM_HOST),
          e.get());
    return ok;
}
inline std::vector<uint8_t> note_sender_decrypt_batch(const JubJubScalar* a, const JubJubScalar* b, size_t n_secret,
                                                      const Scalar* R, const Scalar* note_pk, const Scalar* enc, size_t n,
                                                      const Scalar (&G_uv)[2], std::vector<Scalar>& A,
                                                      std::vector<Scalar>& B, size_t* n_failed = nullptr,
                                                      Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok(n, 0);
    A.assign(2 * n, Scalar{});
    B.assign(2 * n, Scalar{});
    check(p252_note_sender_decrypt_batch(e.get(), a, b, n_secret, R, note_pk, enc, n, G_uv, A.data(), B.data(), ok.data(),
                                         n_failed, P252_MEM_HOST),
          e.get());
    return ok;
}

// NEW: multi-scalar multiplication and all-or-nothing Schnorr batch verification (p252_jubjub_msm /
// p252_schnorr_verify_all).  VARIABLE TIME: scalar bits become bucket indexes on the device, so both take public data only.
// sum [scalars[i]] points[i] over the valid items into out_uv (the identity (0, 1) for n == 0); points holds n x 2
// scalars; an item with a scalar >= r_J, a coordinate >= p or a point off the curve is skipped.  n_invalid may be null.
inline void jubjub_msm(const JubJubScalar* scalars, const Scalar* points, size_t n, Scalar (&out_uv)[2],
                       size_t* n_invalid = nullptr, Engine& e = Engine::default_engine()) {
    check(p252_jubjub_msm(e.get(), scalars, points, n, out_uv, n_invalid, P252_MEM_HOST), e.get());
}
// true iff no item is invalid, every R is on the curve and [8] ([sum z u] G + sum [z c] PK - sum [z] R) is the identity
// (c = challenge(R, m), z = weight): cofactored, so an R shifted by a small-order point passes.  pk holds 1 or n points
// (n_public), R n x 2 scalars; weight holds n caller-chosen random nonzero scalars (128 bits are enough), unpredictable
// to the signers.  A G off the curve throws Error(P252_ERR_INVALID_POINT).  n_invalid may be null.
inline bool schnorr_verify_all(const Scalar* pk, size_t n_public, const JubJubScalar* u, const Scalar* R, const Scalar* msg,
                               const JubJubScalar* weight, size_t n, const Scalar (&base_uv)[2], size_t* n_invalid = nullptr,
                               Engine& e = Engine::default_engine()) {
    uint8_t all = 0;
    check(p252_schnorr_verify_all(e.get(), pk, n_public, u, R, msg, weight, n, base_uv, &all, n_invalid, P252_MEM_HOST),
          e.get());
    return all != 0;
}
// NEW: all-or-nothing verification of double-key signatures (p252_schnorr_verify_double_all).  VARIABLE TIME: public data
// only.  true iff no item is invalid, every R and R' is on the curve and [8] ([sum z u] G + [sum z' u] G' + sum [z c] PK
// + sum [z' c] PK' - sum [z] R - sum [z'] R') is the identity (c = challenge2(R, R', m), z = weight, z' = weight_p):
// cofactored, so an R shifted by a small-order point passes.  pk and pkp hold 1 or n points each (n_public), R and Rp
// n x 2 scalars; weight and weight_p hold n caller-chosen random nonzero scalars each (128 bits are enough), drawn
// independently of each other and unpredictable to the signers.  A G or G' off the curve throws
// Error(P252_ERR_INVALID_POINT).  n_invalid may be null.
inline bool schnorr_verify_double_all(const Scalar* pk, const Scalar* pkp, size_t n_public, const JubJubScalar* u,
                                      const Scalar* R, const Scalar* Rp, const Scalar* msg, const JubJubScalar* weight,
                                      const JubJubScalar* weight_p, size_t n, const Scalar (&G_uv)[2],
                                      const Scalar (&Gp_uv)[2], size_t* n_invalid = nullptr,
                                      Engine& e = Engine::default_engine()) {
    uint8_t all = 0;
    check(p252_schnorr_verify_double_all(e.get(), pk, pkp, n_public, u, R, Rp, msg, weight, weight_p, n, G_uv, Gp_uv, &all,
                                         n_invalid, P252_MEM_HOST),
          e.get());
    return all != 0;
}

// arity-4 tree of Domain::Merkle4 digests; returns the internal levels bottom-up (root last)
inline std::vector<Scalar> merkle4_build(const std::vector<Scalar>& leaves, Engine& e = Engine::default_engine()) {
    size_t n_internal = 0;
    check(p252_merkle4_tree_nodes(leaves.size(), &n_internal, nullptr));
    std::vector<Scalar> nodes(n_internal);
    check(p252_merkle4_build(e.get(), leaves.data(), leaves.size(), nodes.data(), P252_MEM_HOST), e.get());
    return nodes;
}

// Tree of Domain::Merkle2 / Merkle4 digests for arity 2 / 4 (src/hash.rs:22-31), internal levels bottom-up
inline std::vector<Scalar> merkle_build(int arity, const std::vector<Scalar>& leaves, Engine& e = Engine::default_engine()) {
    size_t n_internal = 0;
    check(p252_merkle_tree_nodes(arity, leaves.size(), &n_internal, nullptr));
    std::vector<Scalar> nodes(n_internal);
    check(p252_merkle_build(e.get(), arity, leaves.data(), leaves.size(), nodes.data(), P252_MEM_HOST), e.get());
    return nodes;
}

// Mirror of poseidon-merkle's `Opening<T, H, A>` (consumer crate, AGENTS.md:62-66): the root, for every level
// (0 = leaf level) the whole sibling group of the path node, and the node's offset inside the group.
struct Opening {
    int arity = 4;
    Scalar root{};
    std::vector<Scalar> branch;       // depth x arity
    std::vector<size_t> positions;    // depth
    uint64_t leaf_index = 0;
    size_t depth() const { return positions.size(); }
    // Opening::verify(item): depth chained Merkle digests + membership checks, on the device
    bool verify(const Scalar& item, Engine& e = Engine::default_engine()) const {
        uint8_t ok = 0;
        check(p252_merkle_verify_batch(e.get(), arity, static_cast<int>(depth()), &item, &leaf_index, branch.data(), &root,
                                       1, &ok, nullptr, P252_MEM_HOST),
              e.get());
        return ok != 0;
    }
};

// Openings of the leaves `leaf_idx` of a tree held as leaves + nodes (merkle_build layout)
inline std::vector<Opening> merkle_open_batch(int arity, const std::vector<Scalar>& leaves, const std::vector<Scalar>& nodes,
                                              const std::vector<uint64_t>& leaf_idx, Engine& e = Engine::default_engine()) {
    int depth = 0;
    size_t n_internal = 0;
    check(p252_merkle_tree_nodes(arity, leaves.size(), &n_internal, &depth));
    if (nodes.size() != n_internal) throw Error(P252_ERR_INVALID_ARGUMENT, "node array does not match the leaf count");
    std::vector<Scalar> paths(leaf_idx.size() * depth * arity);
    check(p252_merkle_open_batch(e.get(), arity, leaves.data(), leaves.size(), nodes.data(), leaf_idx.data(), leaf_idx.size(),
                                 paths.data(), P252_MEM_HOST),
          e.get());
    std::vector<Opening> out(leaf_idx.size());
    for (size_t i = 0; i < out.size(); ++i) {
        Opening& o = out[i];
        o.arity = arity;
        o.root = nodes.back();
        o.leaf_index = leaf_idx[i];
        o.branch.assign(paths.begin() + i * depth * arity, paths.begin() + (i + 1) * depth * arity);
        uint64_t idx = leaf_idx[i];
        for (int l = 0; l < depth; ++l, idx /= static_cast<uint64_t>(arity)) o.positions.push_back(idx % arity);
    }
    return out;
}

// Fixed-height tree of poseidon-merkle's `Tree<T, H, A>` shape over p252_mtree (host buffers): room for `capacity`
// <= arity^height leaves; empty slots and empty subtrees are the zero scalar (src/hash.rs:24-26).  `extend` appends,
// `update` overwrites (the last write to a leaf wins); both rehash only the touched paths on the device.
class Tree {
public:
    Tree(int arity, int height, uint64_t capacity, Engine& e = Engine::default_engine()) : e_(&e) {
        uint64_t leaf_slots = 0, node_slots = 0;
        check(p252_mtree_layout(arity, height, capacity, &leaf_slots, &node_slots, nullptr));
        leaves_.assign(leaf_slots, Scalar{});
        nodes_.assign(node_slots, Scalar{});
        t_.struct_size = sizeof(p252_mtree);
        t_.arity = arity;
        t_.height = height;
        t_.reserved = 0;
        t_.capacity = capacity;
        t_.n_leaves = 0;
    }
    void extend(const std::vector<Scalar>& values) { run(nullptr, nullptr, 0, values.data(), values.size()); }
    void update(const std::vector<uint64_t>& idx, const std::vector<Scalar>& values) {
        if (idx.size() != values.size()) throw Error(P252_ERR_INVALID_ARGUMENT, "idx and values differ in length");
        run(idx.data(), values.data(), idx.size(), nullptr, 0);
    }
    const Scalar& root() const { return nodes_.back(); }
    uint64_t size() const { return t_.n_leaves; }
    const std::vector<Scalar>& leaves() const { return leaves_; }
    const std::vector<Scalar>& nodes() const { return nodes_; }
    // the poseidon-merkle `Opening` of leaf i
    Opening opening(uint64_t i) {
        Opening o;
        o.arity = t_.arity;
        o.root = root();
        o.leaf_index = i;
        o.branch.resize((size_t)t_.height * t_.arity);
        check(p252_mtree_open_batch(e_->get(), bind(), &i, 1, o.branch.data(), P252_MEM_HOST), e_->get());
        for (int l = 0; l < t_.height; ++l, i /= (uint64_t)t_.arity) o.positions.push_back(i % t_.arity);
        return o;
    }

private:
    p252_mtree* bind() {
        t_.leaves = leaves_.data();
        t_.nodes = nodes_.data();
        return &t_;
    }
    void run(const uint64_t* idx, const Scalar* values, size_t n_upd, const Scalar* append, size_t n_append) {
        check(p252_mtree_update(e_->get(), bind(), idx, values, n_upd, append, n_append, nullptr, P252_MEM_HOST), e_->get());
    }
    Engine* e_;
    p252_mtree t_{};
    std::vector<Scalar> leaves_, nodes_;
};

// Sparse fixed-height tree over p252_smtree (host buffers): poseidon-merkle's `Tree::insert(pos, item)` and
// `Tree::remove(pos)` at any position below `capacity` <= arity^height.  Empty leaves and nodes with no value below them
// are the zero scalar and are never hashed; a present leaf of value zero is not an empty one.  Batches rehash only the
// touched paths on the device.
class SparseTree {
public:
    SparseTree(int arity, int height, uint64_t capacity, Engine& e = Engine::default_engine()) : e_(&e) {
        uint64_t leaf_slots = 0, node_slots = 0;
        check(p252_mtree_layout(arity, height, capacity, &leaf_slots, &node_slots, nullptr));
        leaves_.assign(leaf_slots, Scalar{});
        nodes_.assign(node_slots, Scalar{});
        present_.assign(leaf_slots + node_slots, 0);
        t_.struct_size = sizeof(p252_smtree);
        t_.arity = arity;
        t_.height = height;
        t_.reserved = 0;
        t_.capacity = capacity;
    }
    // ops[i] == 0 inserts / overwrites values[i] at pos[i], ops[i] == 1 removes pos[i]; as if applied one after another
    void apply(const std::vector<uint64_t>& pos, const std::vector<uint8_t>& ops, const std::vector<Scalar>& values) {
        if (pos.size() != ops.size() || pos.size() != values.size())
            throw Error(P252_ERR_INVALID_ARGUMENT, "pos, ops and values differ in length");
        run(pos, ops.data(), values.data());
    }
    void insert(const std::vector<uint64_t>& pos, const std::vector<Scalar>& values) {
        if (pos.size() != values.size()) throw Error(P252_ERR_INVALID_ARGUMENT, "pos and values differ in length");
        run(pos, nullptr, values.data());
    }
    void remove(const std::vector<uint64_t>& pos) {
        apply(pos, std::vector<uint8_t>(pos.size(), 1), std::vector<Scalar>(pos.size()));
    }
    // recompute every node from the leaves and their presence
    void build() { check(p252_smtree_build(e_->get(), bind(), P252_MEM_HOST), e_->get()); }
    const Scalar& root() const { return nodes_.back(); }
    bool contains(uint64_t pos) const { return pos < t_.capacity && present_[pos] != 0; }
    uint64_t size() {
        uint64_t n = 0;
        check(p252_smtree_len(e_->get(), bind(), &n, P252_MEM_HOST), e_->get());
        return n;
    }
    const std::vector<Scalar>& leaves() const { return leaves_; }
    const std::vector<Scalar>& nodes() const { return nodes_; }
    const std::vector<uint8_t>& present() const { return present_; }
    // the poseidon-merkle `Opening` of the present position pos
    Opening opening(uint64_t pos) {
        Opening o;
        o.arity = t_.arity;
        o.root = root();
        o.leaf_index = pos;
        o.branch.resize((size_t)t_.height * t_.arity);
        check(p252_smtree_open_batch(e_->get(), bind(), &pos, 1, o.branch.data(), P252_MEM_HOST), e_->get());
        for (int l = 0; l < t_.height; ++l, pos /= (uint64_t)t_.arity) o.positions.push_back(pos % t_.arity);
        return o;
    }

private:
    p252_smtree* bind() {
        t_.leaves = leaves_.data();
        t_.nodes = nodes_.data();
        t_.present = present_.data();
        return &t_;
    }
    void run(const std::vector<uint64_t>& pos, const uint8_t* ops, const Scalar* values) {
        check(p252_smtree_update(e_->get(), bind(), pos.data(), ops, values, pos.size(), nullptr, P252_MEM_HOST), e_->get());
    }
    Engine* e_;
    p252_smtree t_{};
    std::vector<Scalar> leaves_, nodes_;
    std::vector<uint8_t> present_;
};

// Compact sparse tree over p252_ctree (host buffers): poseidon-merkle's `Tree<T, H, A>` at any height, positions anywhere
// below arity^height (every u64 at arity 2 / height 64 or arity 4 / height 32), storage proportional to at most
// `max_leaves` present positions.  Each level is the sorted list of its present nodes; presence and the empty-subtree
// rule are those of SparseTree.
class CompactTree {
public:
    CompactTree(int arity, int height, uint64_t max_leaves, Engine& e = Engine::default_engine()) : e_(&e) {
        uint64_t total = 0;
        offset_.resize((size_t)(height > 0 && height <= 64 ? height : 0) + 1);
        check(p252_ctree_layout(arity, height, max_leaves, &total, offset_.data()));
        keys_.assign(total, 0);
        values_.assign(total, Scalar{});
        count_.assign((size_t)height + 1, 0);
        t_.struct_size = sizeof(p252_ctree);
        t_.arity = arity;
        t_.height = height;
        t_.reserved = 0;
        t_.max_leaves = max_leaves;
    }
    // ops[i] == 0 inserts / overwrites values[i] at pos[i], ops[i] == 1 removes pos[i]; as if applied one after another
    void apply(const std::vector<uint64_t>& pos, const std::vector<uint8_t>& ops, const std::vector<Scalar>& values) {
        if (pos.size() != ops.size() || pos.size() != values.size())
            throw Error(P252_ERR_INVALID_ARGUMENT, "pos, ops and values differ in length");
        run(pos, ops.data(), values.data());
    }
    void insert(const std::vector<uint64_t>& pos, const std::vector<Scalar>& values) {
        if (pos.size() != values.size()) throw Error(P252_ERR_INVALID_ARGUMENT, "pos and values differ in length");
        run(pos, nullptr, values.data());
    }
    void remove(const std::vector<uint64_t>& pos) {
        apply(pos, std::vector<uint8_t>(pos.size(), 1), std::vector<Scalar>(pos.size()));
    }
    const Scalar& root() const { return values_[offset_.back()]; }
    uint64_t size() const { return count_[0]; }
    bool contains(uint64_t pos) const {
        const auto end = keys_.begin() + (std::ptrdiff_t)count_[0];
        const auto it = std::lower_bound(keys_.begin(), end, pos);
        return it != end && *it == pos;
    }
    const std::vector<uint64_t>& keys() const { return keys_; }
    const std::vector<Scalar>& values() const { return values_; }
    const std::vector<uint64_t>& count() const { return count_; }
    const std::vector<uint64_t>& level_offset() const { return offset_; }
    // the poseidon-merkle `Opening` of the present position pos
    Opening opening(uint64_t pos) {
        Opening o;
        o.arity = t_.arity;
        o.root = root();
        o.leaf_index = pos;
        o.branch.resize((size_t)t_.height * t_.arity);
        check(p252_ctree_open_batch(e_->get(), bind(), &pos, 1, o.branch.data(), P252_MEM_HOST), e_->get());
        for (int l = 0; l < t_.height; ++l, pos /= (uint64_t)t_.arity) o.positions.push_back(pos % t_.arity);
        return o;
    }

private:
    p252_ctree* bind() {
        t_.keys = keys_.data();
        t_.values = values_.data();
        t_.count = count_.data();
        return &t_;
    }
    void run(const std::vector<uint64_t>& pos, const uint8_t* ops, const Scalar* values) {
        check(p252_ctree_update(e_->get(), bind(), pos.data(), ops, values, pos.size(), nullptr, P252_MEM_HOST), e_->get());
    }
    Engine* e_;
    p252_ctree t_{};
    std::vector<uint64_t> keys_, count_, offset_;
    std::vector<Scalar> values_;
};

// n x Opening::verify with all openings in one launch: ok[i] != 0 iff paths[i] proves items[i] under root
inline std::vector<uint8_t> merkle_verify_batch(int arity, int depth, const Scalar* items, const uint64_t* leaf_idx,
                                                const Scalar* paths, const Scalar& root, size_t n,
                                                Engine& e = Engine::default_engine()) {
    std::vector<uint8_t> ok(n);
    check(p252_merkle_verify_batch(e.get(), arity, depth, items, leaf_idx, paths, &root, n, ok.data(), nullptr, P252_MEM_HOST),
          e.get());
    return ok;
}

}  // namespace p252
