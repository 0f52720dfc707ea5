/*
 * randomx_oracle.h — CPU ORACLE for k2pow (RandomX).  TEST INFRASTRUCTURE ONLY: only tests/, smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it; the product (libb200post.so) never links or calls it.
 * See randomx_oracle.c for what it restates and how it is pinned.
 */
#ifndef RANDOMX_ORACLE_H
#define RANDOMX_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct rxo_ss_instr { uint8_t opcode, dst, src, mod; uint32_t imm32; uint64_t rcp; } rxo_ss_instr;
typedef struct rxo_ss_program { rxo_ss_instr ins[512]; uint32_t size, address_reg; } rxo_ss_program;
typedef struct rxo_cache rxo_cache;
typedef struct rxo_vm rxo_vm;

/* primitives */
void rxo_blake2b(void *out, size_t outlen, const void *in, size_t inlen);
int rxo_argon2d_fill(uint64_t *mem, uint32_t m_blocks, uint32_t t_cost, const void *pwd, uint32_t pwdlen,
                     const void *salt, uint32_t saltlen, uint32_t taglen, uint8_t *tag);
void rxo_soft_aesenc(uint8_t st[16], const uint8_t key[16]);
void rxo_soft_aesdec(uint8_t st[16], const uint8_t key[16]);
void rxo_set_soft_aes(int on);
int rxo_has_aesni(void);
void rxo_aes_constants(uint8_t gen1r[64], uint8_t gen4r[128], uint8_t hash_state[64], uint8_t hash_xkeys[32]);
void rxo_fill_aes_1rx4(uint8_t state[64], size_t outlen, uint8_t *out);
void rxo_fill_aes_4rx4(const uint8_t state[64], size_t outlen, uint8_t *out);
void rxo_hash_aes_1rx4(const uint8_t *in, size_t inlen, uint8_t out[64]);
uint64_t rxo_reciprocal(uint32_t divisor);
void rxo_opcode_map(uint8_t out[256]);

/* cache (256 MiB Argon2d memory + 8 SuperscalarHash programs), dataset items, optional full dataset (2080 MiB) */
rxo_cache *rxo_cache_new(const void *key, size_t keylen);
void rxo_cache_free(rxo_cache *c);
const uint64_t *rxo_cache_memory(const rxo_cache *c);
const rxo_ss_program *rxo_cache_programs(const rxo_cache *c);
void rxo_dataset_item(const rxo_cache *c, uint64_t item, uint64_t out[8]);
int rxo_dataset_init(rxo_cache *c, int threads);
int rxo_has_dataset(const rxo_cache *c);
/* the fast-mode dataset (34 078 719 items x 64 bytes, after rxo_dataset_init), or NULL if there is none */
const uint8_t *rxo_dataset_memory(const rxo_cache *c);

/* the hash */
rxo_vm *rxo_vm_new(void);
void rxo_vm_free(rxo_vm *v);
void rxo_hash_vm(rxo_vm *v, const rxo_cache *cache, const void *input, size_t inlen, uint8_t out[32], uint8_t *trace);
void rxo_hash(const rxo_cache *cache, const void *input, size_t inlen, uint8_t out[32]);

/* k2pow */
void rxo_k2pow_input(uint64_t pow, uint8_t nonce_group, const uint8_t challenge8[8], const uint8_t node_id[32], uint8_t out[48]);
double rxo_k2pow_scan(const rxo_cache *cache, uint8_t nonce_group, const uint8_t challenge8[8], const uint8_t node_id[32],
                      const uint8_t *difficulty, uint64_t start, uint64_t count, int threads, uint8_t *hashes, uint64_t *found_pow);

#ifdef __cplusplus
}
#endif
#endif
