// modes_tables.h — host-side construction of the constant tables the kernels use.
// Behavioural references (reference tree): convert.c:35-62 (UC8 magnitude table),
// crc.c:42-82 (CRC-24, generator 0xFFF409), crc.c:180-378 (single-bit error syndromes).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "common.h"

// Full 65536-entry table, index = I*256 + Q.  The arithmetic has to round exactly like the
// reference's: (x-127.5)/127.5 in double narrowed to float, float multiply and add rounded
// separately (no FMA), correctly rounded sqrtf, then *65535 + 0.5 truncated.
static inline void b200_build_uc8_lut(uint16_t *lut) {
    float f[256];
    for (int i = 0; i < 256; i++) f[i] = (float)(((double)i - 127.5) / 127.5);
    for (int i = 0; i < 256; i++) {
        volatile float fi2 = f[i] * f[i];           // volatile: keep the two products and the sum
        for (int q = 0; q < 256; q++) {             // as separate IEEE single operations
            volatile float fq2 = f[q] * f[q];
            volatile float magsq = fi2 + fq2;
            float ms = magsq > 1.0f ? 1.0f : magsq;
            volatile float mag = sqrtf(ms);
            volatile float scaled = mag * 65535.0f;
            volatile float biased = scaled + 0.5f;
            lut[i * 256 + q] = (uint16_t)biased;
        }
    }
}

static inline uint32_t b200_crc32_ieee(const void *data, size_t n) {
    const uint8_t *p = (const uint8_t *)data;
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xedb88320u & (0u - (c & 1u)));
    }
    return ~c;
}

// Folded table: the magnitude depends only on |2I-255| and |2Q-255|, so 128 x 128 entries suffice.
// fold(v) = v >= 128 ? 255 - v : v  (127 = centre, 0 = full scale: `(v ^ sign) & 0x7f` on the device, a single LOP3 for four
// bytes).  Entry (fi, fq) is stored at uint16 index
//   fq*128 + (fi ^ ((fq & 15) << 2))
// i.e. byte offset fq*256 + 2*fi with bits 3..6 XOR-ed by (fq & 15): rows that differ in their low
// four bits land in different shared-memory banks, which matters because receiver noise keeps
// almost all lookups inside a tiny corner of the table.
static inline void b200_build_folded_lut(const uint16_t *lut_full, uint16_t *fold) {
    for (int fq = 0; fq < 128; fq++)
        for (int fi = 0; fi < 128; fi++)
            fold[fq * 128 + (fi ^ ((fq & 15) << 2))] = lut_full[fi * 256 + fq];
}

static inline uint32_t b200_crc24_bytes(const uint32_t *tab, const uint8_t *msg, int nbytes) {
    uint32_t rem = 0;
    for (int i = 0; i < nbytes - 3; i++) rem = ((rem << 8) ^ tab[msg[i] ^ ((rem >> 16) & 0xff)]) & 0xffffffu;
    return rem ^ ((uint32_t)msg[nbytes - 3] << 16) ^ ((uint32_t)msg[nbytes - 2] << 8) ^ msg[nbytes - 1];
}

// Returns 0 on success.  syn_hash is a perfect hash of the 112 single-bit syndromes:
// slot = (syndrome * mul) >> 23 (9 bits); entry = syndrome << 8 | bit, 0 when empty.  (An empty slot must not look like any
// syndrome a lookup can ask for: with 0xffffffff as the marker the syndrome 0xffffff "matched" empty slots and came back as a
// correctable error in bit 255 — found by tools/emu_fuzz.py.  Entry 0 can only match syndrome 0, which reports bit 0: never
// correctable, crc.c:210-211.)
static inline int b200_build_tables(DeviceTables *t, uint16_t *lut_full /*65536*/) {
    b200_build_uc8_lut(lut_full);
    b200_build_folded_lut(lut_full, t->lut_fold);
    for (int i = 0; i < 256; i++) {
        uint32_t c = (uint32_t)i << 16;
        for (int j = 0; j < 8; j++) c = (c & 0x800000u) ? ((c << 1) ^ 0xfff409u) : (c << 1);
        t->crc_tab[i] = c & 0xffffffu;
    }
    for (int b = 0; b < 112; b++) {
        uint8_t m[14];
        memset(m, 0, sizeof m);
        m[b >> 3] = (uint8_t)(1u << (7 - (b & 7)));
        t->bit_syn[b] = b200_crc24_bytes(t->crc_tab, m, 14);
    }
    for (uint32_t mul = 0x9E3779B1u, tries = 0; tries < 200000; tries++, mul += 0x61C88646u) {
        uint32_t m = mul | 1u;
        memset(t->syn_hash, 0, sizeof t->syn_hash);
        int ok = 1;
        for (int b = 0; b < 112 && ok; b++) {
            uint32_t h = (t->bit_syn[b] * m) >> 23;
            if (t->syn_hash[h] != 0u) ok = 0;
            else t->syn_hash[h] = (t->bit_syn[b] << 8) | (uint32_t)b;
        }
        if (ok) { t->syn_hash_mul = m; return 0; }
    }
    return -1;
}
