/* roaring_check.c — a second, independent restatement of rb_build_agg's bytes (CRoaring v0.2.66: add(), runOptimize(), portable
 * serialization), for tests/test_rb_plan.py to cross-check tests/roaring_oracle.py against.  Where the Python oracle works on sorted
 * arrays, this one keeps every container as a 65536-bit bitset and counts cardinality and runs the way CRoaring's bitset container
 * does (popcount; a run ends at every set bit whose successor is clear).
 *
 * stdin:  repeated { uint32 n; uint32 values[n] }  (any order, duplicates allowed)
 * stdout: repeated { uint32 bytes; uint8 serialized[bytes] } */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

enum { T_ARRAY = 1, T_BITSET = 2, T_RUN = 3 };

typedef struct { uint16_t key; uint32_t card, runs; int type; uint64_t* bits; } Cont;

static int cmp_u32(const void* a, const void* b) { uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b; return x < y ? -1 : x > y; }

static void put(uint8_t** o, uint64_t v, int n) { for (int i = 0; i < n; i++) *(*o)++ = (uint8_t)(v >> (8 * i)); }

static size_t payload_bytes(const Cont* c) { return c->type == T_ARRAY ? 2u * c->card : c->type == T_RUN ? 2u + 4u * c->runs : 8192u; }

int main(void) {
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        uint32_t* v = (uint32_t*)malloc((size_t)(n ? n : 1) * 4);
        if (n && fread(v, 4, n, stdin) != n) return 2;
        qsort(v, n, 4, cmp_u32);
        Cont* cs = (Cont*)calloc(n ? n : 1, sizeof(Cont));
        uint32_t size = 0;
        for (uint32_t i = 0; i < n; i++) {
            const uint16_t key = (uint16_t)(v[i] >> 16);
            if (size == 0 || cs[size - 1].key != key) { cs[size].key = key; cs[size].bits = (uint64_t*)calloc(1024, 8); size++; }
            cs[size - 1].bits[(v[i] & 0xFFFF) >> 6] |= 1ull << (v[i] & 63);
        }
        int has_run = 0;
        size_t total = 0;
        for (uint32_t c = 0; c < size; c++) {
            Cont* x = &cs[c];
            for (int w = 0; w < 1024; w++) {
                x->card += (uint32_t)__builtin_popcountll(x->bits[w]);
                const uint64_t next = w < 1023 ? x->bits[w + 1] & 1 : 0;   /* bit 0 of the next word follows bit 63 */
                x->runs += (uint32_t)__builtin_popcountll(x->bits[w] & ~((x->bits[w] >> 1) | (next << 63)));
            }
            /* add(): ARRAY up to DEFAULT_MAX_SIZE (4096), then BITSET; runOptimize(): RUN when strictly smaller serialized */
            if (x->card <= 4096) x->type = (2 + 4 * x->runs < 2 + 2 * x->card) ? T_RUN : T_ARRAY;
            else x->type = (2 + 4 * x->runs < 8192) ? T_RUN : T_BITSET;
            has_run |= x->type == T_RUN;
            total += payload_bytes(x);
        }
        const uint32_t nrb = (size + 7) / 8;
        const int offsets = !has_run || size >= 4;
        const size_t hdr = has_run ? 4 + nrb + 4 * (size_t)size + (offsets ? 4 * (size_t)size : 0) : 8 + 8 * (size_t)size;
        uint8_t* buf = (uint8_t*)calloc(hdr + total + 1, 1);
        uint8_t* o = buf;
        if (has_run) {
            put(&o, 12347u | ((size - 1) << 16), 4);
            for (uint32_t c = 0; c < size; c++) if (cs[c].type == T_RUN) o[c / 8] |= (uint8_t)(1u << (c % 8));
            o += nrb;
        } else { put(&o, 12346u, 4); put(&o, size, 4); }
        for (uint32_t c = 0; c < size; c++) { put(&o, cs[c].key, 2); put(&o, cs[c].card - 1, 2); }
        if (offsets) {
            uint32_t off = (uint32_t)hdr;
            for (uint32_t c = 0; c < size; c++) { put(&o, off, 4); off += (uint32_t)payload_bytes(&cs[c]); }
        }
        for (uint32_t c = 0; c < size; c++) {
            const Cont* x = &cs[c];
            if (x->type == T_BITSET) { for (int w = 0; w < 1024; w++) put(&o, x->bits[w], 8); continue; }
            if (x->type == T_RUN) put(&o, x->runs, 2);
            for (int b = 0; b < 65536;) {
                if (!((x->bits[b >> 6] >> (b & 63)) & 1)) { b++; continue; }
                if (x->type == T_ARRAY) { put(&o, (uint64_t)b, 2); b++; continue; }
                int e = b;
                while (e + 1 < 65536 && ((x->bits[(e + 1) >> 6] >> ((e + 1) & 63)) & 1)) e++;
                put(&o, (uint64_t)b, 2); put(&o, (uint64_t)(e - b), 2);
                b = e + 1;
            }
        }
        const uint32_t len = (uint32_t)(o - buf);
        if (len != hdr + total) return 3;
        fwrite(&len, 4, 1, stdout);
        fwrite(buf, 1, len, stdout);
        for (uint32_t c = 0; c < size; c++) free(cs[c].bits);
        free(cs); free(buf); free(v);
    }
    return 0;
}
