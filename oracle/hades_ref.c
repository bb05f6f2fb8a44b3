/* CPU ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C restatement of the dusk-poseidon hot path with the SAME dense algorithm and the SAME
 * in-memory representation as the reference (BlsScalar = 4 x u64 LE limbs, Montgomery form,
 * R = 2^256 mod p): ARC -> x^5 as two squarings and one multiply -> dense 25-multiply MDS.
 * No algebraic shortcut.  It is (a) the fast checker for the CUDA path at sizes the Python
 * oracle (hades_oracle.py) is too slow for, and (b) the timed CPU baseline
 * ("port": the Rust reference cannot be built here -- no cargo/rustc, deps not vendored).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  The product (poseidon252_b200/) never links or calls it.
 *
 * Pinned by: tests/test_oracle.py checks this file against hades_oracle.py, which reproduces the
 * 6 known-answer vectors of src/hades.rs:134-162.
 * Parity unpinned: tag derivation (not done here: the tag is an input scalar) -- see
 * hades_oracle.py header.
 *
 * Reference lines restated (relative to the reference repository's root):
 *   src/hades/permutation.rs:63-72,83-92,105-123   round schedule
 *   src/hades/permutation/scalar.rs:39-64          add_round_constants, quintic_s_box, mul_matrix
 *   src/hades/round_constants.rs:40-47, src/hades/mds_matrix.rs:25-32   from_raw of file limbs
 *   dusk-safe 0.3 Sponge (driven at src/hash.rs:128-155; src/encryption.rs:62-95)
 */
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "hades_constants.h"

typedef unsigned __int128 u128;
typedef struct { uint64_t l[4]; } fr;

#define WIDTH 5
#define FULL_ROUNDS 8
#define PARTIAL_ROUNDS 60
#define ROUNDS (FULL_ROUNDS + PARTIAL_ROUNDS)
#define RATE 4

static const uint64_t MOD[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL,
                                0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
static const uint64_t INV = 0xfffffffeffffffffULL; /* -p^-1 mod 2^64 */
static const fr R2 = {{0xc999e990f3f29c6dULL, 0x2b6cedcb87925c23ULL, 0x05d314967254398fULL,
                       0x0748d9d99f59ff11ULL}};

static fr ARC[ROUNDS][WIDTH]; /* Montgomery form of ROUND_CONSTANTS[round][i] */
static fr MDS[WIDTH][WIDTH];  /* Montgomery form of MDS_MATRIX[i][j]          */
static int g_init = 0;

/* r = a - p if a >= p (a < 2p) */
static inline void fr_cond_sub(fr *a) {
    uint64_t t[4];
    u128 b = 0;
    for (int i = 0; i < 4; i++) {
        u128 d = (u128)a->l[i] - MOD[i] - (uint64_t)b;
        t[i] = (uint64_t)d;
        b = (d >> 64) & 1;
    }
    if (!b) memcpy(a->l, t, sizeof t);
}

/* BlsScalar + (dusk-bls12_381 Scalar::add) */
static inline fr fr_add(const fr *a, const fr *b) {
    fr r;
    u128 c = 0;
    for (int i = 0; i < 4; i++) {
        c += (u128)a->l[i] + b->l[i];
        r.l[i] = (uint64_t)c;
        c >>= 64;
    }
    /* p < 2^255, so a+b < 2^256: no carry out */
    fr_cond_sub(&r);
    return r;
}

/* BlsScalar - */
static inline fr fr_sub(const fr *a, const fr *b) {
    fr r;
    u128 bw = 0;
    for (int i = 0; i < 4; i++) {
        u128 d = (u128)a->l[i] - b->l[i] - (uint64_t)bw;
        r.l[i] = (uint64_t)d;
        bw = (d >> 64) & 1;
    }
    if (bw) {
        u128 c = 0;
        for (int i = 0; i < 4; i++) {
            c += (u128)r.l[i] + MOD[i];
            r.l[i] = (uint64_t)c;
            c >>= 64;
        }
    }
    return r;
}

/* BlsScalar * : Montgomery product a*b/R mod p, fully reduced (CIOS, 64-bit digits) */
static inline fr fr_mul(const fr *a, const fr *b) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        u128 c = 0;
        for (int j = 0; j < 4; j++) {
            c += (u128)a->l[j] * b->l[i] + t[j];
            t[j] = (uint64_t)c;
            c >>= 64;
        }
        c += t[4];
        t[4] = (uint64_t)c;
        t[5] = (uint64_t)(c >> 64);
        uint64_t m = t[0] * INV;
        c = (u128)m * MOD[0] + t[0];
        c >>= 64;
        for (int j = 1; j < 4; j++) {
            c += (u128)m * MOD[j] + t[j];
            t[j - 1] = (uint64_t)c;
            c >>= 64;
        }
        c += t[4];
        t[3] = (uint64_t)c;
        t[4] = t[5] + (uint64_t)(c >> 64);
    }
    fr r = {{t[0], t[1], t[2], t[3]}};
    fr_cond_sub(&r);
    return r;
}

static inline int fr_eq(const fr *a, const fr *b) { return memcmp(a->l, b->l, 32) == 0; }

void oracle_init(void) {
    if (g_init) return;
    for (int r = 0; r < ROUNDS; r++)
        for (int i = 0; i < WIDTH; i++) {
            fr raw;
            memcpy(raw.l, ORACLE_ARC_RAW[r * WIDTH + i], 32);
            ARC[r][i] = fr_mul(&raw, &R2); /* BlsScalar::from_raw */
        }
    for (int i = 0; i < WIDTH; i++)
        for (int j = 0; j < WIDTH; j++) {
            fr raw;
            memcpy(raw.l, ORACLE_MDS_RAW[i * WIDTH + j], 32);
            MDS[i][j] = fr_mul(&raw, &R2);
        }
    g_init = 1;
}

/* src/hades/permutation/scalar.rs:39-48 */
static inline void add_round_constants(int round, fr *s) {
    for (int i = 0; i < WIDTH; i++) s[i] = fr_add(&s[i], &ARC[round][i]);
}
/* src/hades/permutation/scalar.rs:50-52 */
static inline void quintic_s_box(fr *v) {
    fr v2 = fr_mul(v, v);
    fr v4 = fr_mul(&v2, &v2);
    *v = fr_mul(&v4, v);
}
/* src/hades/permutation/scalar.rs:54-64 */
static inline void mul_matrix(fr *s) {
    fr result[WIDTH];
    memset(result, 0, sizeof result);
    for (int j = 0; j < WIDTH; j++)
        for (int k = 0; k < WIDTH; k++) {
            fr t = fr_mul(&MDS[k][j], &s[j]);
            result[k] = fr_add(&result[k], &t);
        }
    memcpy(s, result, sizeof result);
}
/* src/hades/permutation.rs:105-123 */
static void perm(fr *s) {
    for (int r = 0; r < FULL_ROUNDS / 2; r++) {
        add_round_constants(r, s);
        for (int i = 0; i < WIDTH; i++) quintic_s_box(&s[i]);
        mul_matrix(s);
    }
    for (int r = 0; r < PARTIAL_ROUNDS; r++) {
        add_round_constants(r + FULL_ROUNDS / 2, s);
        quintic_s_box(&s[WIDTH - 1]);
        mul_matrix(s);
    }
    for (int r = 0; r < FULL_ROUNDS / 2; r++) {
        add_round_constants(r + FULL_ROUNDS / 2 + PARTIAL_ROUNDS, s);
        for (int i = 0; i < WIDTH; i++) quintic_s_box(&s[i]);
        mul_matrix(s);
    }
}

/* ---- sponge (dusk-safe 0.3 schedule; see hades_oracle.py Sponge) ---- */
typedef struct {
    fr state[WIDTH];
    int pos_absorb, pos_squeeze;
} sponge_t;

static inline void sponge_start(sponge_t *sp, const fr *tag) {
    memset(sp, 0, sizeof *sp);
    sp->state[0] = *tag;
}
static inline void sponge_absorb(sponge_t *sp, const fr *in, size_t n) {
    for (size_t k = 0; k < n; k++) {
        if (sp->pos_absorb == RATE) {
            perm(sp->state);
            sp->pos_absorb = 0;
        }
        int pos = sp->pos_absorb + 1;
        sp->state[pos] = fr_add(&sp->state[pos], &in[k]);
        sp->pos_absorb++;
    }
    sp->pos_squeeze = RATE;
}
static inline void sponge_squeeze(sponge_t *sp, fr *out, size_t n) {
    for (size_t k = 0; k < n; k++) {
        if (sp->pos_squeeze == RATE) {
            perm(sp->state);
            sp->pos_squeeze = 0;
            sp->pos_absorb = 0;
        }
        out[k] = sp->state[sp->pos_squeeze + 1];
        sp->pos_squeeze++;
    }
}

/* ---- single-thread entry points (all buffers: item-major arrays of BlsScalar.0 limbs) ---- */
void oracle_permute(fr *states, size_t n) {
    oracle_init();
    for (size_t i = 0; i < n; i++) perm(&states[i * WIDTH]);
}

/* Hash::digest-shaped sponge: Absorb(in_len) ... Squeeze(out_len) with a given tag
 * (src/hash.rs:128-155; chunking of update() only changes the tag, not the schedule). */
void oracle_digest(const fr *tag, const fr *in, size_t n, size_t in_len, fr *out, size_t out_len) {
    oracle_init();
    for (size_t i = 0; i < n; i++) {
        sponge_t sp;
        sponge_start(&sp, tag);
        sponge_absorb(&sp, &in[i * in_len], in_len);
        sponge_squeeze(&sp, &out[i * out_len], out_len);
    }
}

/* KAT-shaped sponge: Absorb(in_len), Absorb(1) of `pad`, Squeeze(1) (src/hades.rs:107-125) */
void oracle_digest_padded(const fr *tag, const fr *in, size_t n, size_t in_len, const fr *pad,
                          fr *out) {
    oracle_init();
    for (size_t i = 0; i < n; i++) {
        sponge_t sp;
        sponge_start(&sp, tag);
        sponge_absorb(&sp, &in[i * in_len], in_len);
        sponge_absorb(&sp, pad, 1);
        sponge_squeeze(&sp, &out[i], 1);
    }
}

/* src/encryption.rs:62-74 -> dusk_safe::encrypt */
void oracle_encrypt(const fr *tag, const fr *msg, size_t n, size_t L, const fr *secret_uv,
                    const fr *nonce, fr *cipher) {
    oracle_init();
    fr *ks = (fr *)malloc((L + 1) * sizeof(fr));
    for (size_t i = 0; i < n; i++) {
        sponge_t sp;
        sponge_start(&sp, tag);
        sponge_absorb(&sp, &secret_uv[i * 2], 2);
        sponge_absorb(&sp, &nonce[i], 1);
        sponge_squeeze(&sp, ks, L);
        sponge_absorb(&sp, &msg[i * L], L);
        sponge_squeeze(&sp, &ks[L], 1);
        for (size_t k = 0; k < L; k++) cipher[i * (L + 1) + k] = fr_add(&msg[i * L + k], &ks[k]);
        cipher[i * (L + 1) + L] = ks[L];
    }
    free(ks);
}

/* src/encryption.rs:83-95 -> dusk_safe::decrypt; ok[i] = 0 <=> Error::DecryptionFailed */
void oracle_decrypt(const fr *tag, const fr *cipher, size_t n, size_t L, const fr *secret_uv,
                    const fr *nonce, fr *msg, uint8_t *ok) {
    oracle_init();
    fr *ks = (fr *)malloc((L + 1) * sizeof(fr));
    for (size_t i = 0; i < n; i++) {
        sponge_t sp;
        sponge_start(&sp, tag);
        sponge_absorb(&sp, &secret_uv[i * 2], 2);
        sponge_absorb(&sp, &nonce[i], 1);
        sponge_squeeze(&sp, ks, L);
        for (size_t k = 0; k < L; k++) msg[i * L + k] = fr_sub(&cipher[i * (L + 1) + k], &ks[k]);
        sponge_absorb(&sp, &msg[i * L], L);
        sponge_squeeze(&sp, &ks[L], 1);
        ok[i] = (uint8_t)fr_eq(&ks[L], &cipher[i * (L + 1) + L]);
    }
    free(ks);
}

/* ---- multi-thread wrappers over independent items (the reference itself has no threads;
 *      used only for the reported CPU baseline on all host cores) ---- */
typedef struct {
    int kind; /* 0 = permute, 1 = digest */
    const fr *tag;
    fr *states;
    const fr *in;
    fr *out;
    size_t lo, hi, in_len, out_len;
} job_t;

static void *worker(void *arg) {
    job_t *j = (job_t *)arg;
    if (j->kind == 0)
        oracle_permute(j->states + j->lo * WIDTH, j->hi - j->lo);
    else
        oracle_digest(j->tag, j->in + j->lo * j->in_len, j->hi - j->lo, j->in_len,
                      j->out + j->lo * j->out_len, j->out_len);
    return NULL;
}

static void run_mt(job_t proto, size_t n, int threads) {
    oracle_init();
    if (threads < 1) threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * threads);
    for (int t = 0; t < threads; t++) {
        jobs[t] = proto;
        jobs[t].lo = n * (size_t)t / threads;
        jobs[t].hi = n * (size_t)(t + 1) / threads;
        pthread_create(&th[t], NULL, worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    free(th);
    free(jobs);
}

void oracle_permute_mt(fr *states, size_t n, int threads) {
    job_t j;
    memset(&j, 0, sizeof j);
    j.kind = 0;
    j.states = states;
    run_mt(j, n, threads);
}

void oracle_digest_mt(const fr *tag, const fr *in, size_t n, size_t in_len, fr *out,
                      size_t out_len, int threads) {
    job_t j;
    memset(&j, 0, sizeof j);
    j.kind = 1;
    j.tag = tag;
    j.in = in;
    j.out = out;
    j.in_len = in_len;
    j.out_len = out_len;
    run_mt(j, n, threads);
}

/* field helpers exposed for tests (Montgomery-form in, Montgomery-form out) */
void oracle_fr_mul(const fr *a, const fr *b, fr *r) { *r = fr_mul(a, b); }
void oracle_fr_add(const fr *a, const fr *b, fr *r) { *r = fr_add(a, b); }
void oracle_fr_sub(const fr *a, const fr *b, fr *r) { *r = fr_sub(a, b); }
