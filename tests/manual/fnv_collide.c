// fnv_collide.c - collisions of the 64-bit FNV-1a keys the device path compares before it compares bytes.
//
// A parallel rho search with distinguished points (van Oorschot-Wiener): every trail starts at a point derived from the seed and
// its index, steps x -> f(x) until x has its low D bits zero, and the distinguished point is kept with the trail's start.  Two
// trails that end on one point merged somewhere; walking them again from their starts finds the two inputs with one output.
// Trails are computed in rounds on all threads and merged in index order, so one seed always gives the same pair.
//
//   fnv_collide name [PREFIX]      names PREFIX + 11 chars of [0-9A-Za-z] with one FNV-1a 64.  With PREFIX a name of an earlier
//                                  pair, the two pairs make a 4-way multicollision {a,b} x {c,d} (FNV-1a keeps a collision when the
//                                  same bytes follow).  About half a minute on 8 cores.
//   fnv_collide claw [PREFIX]      a QNAME q and an RNAME r with fnv(q) == fnv(r) ^ 0x9E3779B97F4A7C15 (the filter's RNAME domain):
//                                  one intern slot, two kinds.
//   fnv_collide sig BITS ANCHOR [EXTRA]
//                                  two alleles ANCHOR + 30 bases (BITS 4: 60 bits decide make_sig) or ANCHOR + 28 bases (BITS 8:
//                                  56 bits) with one make_sig; with EXTRA the second allele is EXTRA bases longer (an 'A' tail).
//   options (first): -s SEED (default 1), -t THREADS (default: online CPUs)
//
// Build: gcc -O3 -pthread -o fnv_collide tests/manual/fnv_collide.c
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#define FNV_BASIS 14695981039346656037ull
#define FNV_PRIME 1099511628211ull
#define REF_DOMAIN 0x9E3779B97F4A7C15ull

enum { M_NAME, M_CLAW, M_SIG };
static int mode, bits = 64, sig_bits, extra;
static uint64_t mask, prefix_state = FNV_BASIS, seed = 1;
static char prefix[256], anchor = 'A';
static const char ALPHA[] = "0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz";

static uint64_t splitmix(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// name suffix of x: 11 base-62 digits (62^11 > 2^64)
static void name_of(uint64_t x, char* s) {
    for (int i = 0; i < 11; ++i) { s[i] = ALPHA[x % 62]; x /= 62; }
    s[11] = 0;
}

// allele of x: the anchor, then 2 bits of x per base; the odd branch of a length pair gets `extra` more bases.
static int allele_of(uint64_t x, char* s) {
    static const char B[] = "ACGT";
    const int nb = sig_bits / 2;
    int n = 0;
    s[n++] = anchor;
    for (int i = 0; i < nb; ++i) s[n++] = B[(x >> (2 * i)) & 3];
    if (extra && (x & 1))
        for (int i = 0; i < extra; ++i) s[n++] = 'A';
    s[n] = 0;
    return n;
}

static uint64_t sym(char c) {       // 4-bit mode: the BAM codes A=1 C=2 G=4 T=8; 8-bit mode: the byte
    if (sig_bits == 56) return (uint64_t)(unsigned char)c;
    return c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 4 : 8;
}

// make_sig (polish_dev.cuh) of an allele longer than the exact limit: FNV-1a over the symbols, xor the length, shifted left by 4 / 8.
static uint64_t make_sig(const char* s, int n) {
    uint64_t h = FNV_BASIS;
    for (int i = 0; i < n; ++i) h = (h ^ sym(s[i])) * FNV_PRIME;
    h ^= (uint64_t)n;
    return h << (sig_bits == 60 ? 4 : 8);
}

static uint64_t fnv_from(uint64_t h, const char* s) {
    for (; *s; ++s) h = (h ^ (unsigned char)*s) * FNV_PRIME;
    return h;
}

static uint64_t f(uint64_t x) {
    if (mode == M_SIG) {
        char s[128];
        const int n = allele_of(x, s);
        return (make_sig(s, n) >> (64 - sig_bits)) & mask;
    }
    char s[16];
    name_of(x, s);
    const uint64_t h = fnv_from(prefix_state, s);
    return (mode == M_CLAW && !(x & 1)) ? h ^ REF_DOMAIN : h;
}

// Two inputs collide usefully: different, and for a claw / a length pair, one of each branch.
static int useful(uint64_t a, uint64_t b) {
    if (a == b) return 0;
    if (mode == M_CLAW || (mode == M_SIG && extra)) return ((a ^ b) & 1) != 0;
    return 1;
}

typedef struct { uint64_t start, dp, len; } Trail;
static int dbits;
static uint64_t max_len;
static Trail* round_out;
static uint64_t round_base, round_n;
static volatile uint64_t next_trail;
static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;

static void* worker(void* arg) {
    (void)arg;
    const uint64_t dmask = (1ull << dbits) - 1;
    for (;;) {
        pthread_mutex_lock(&mu);
        const uint64_t i = next_trail++;
        pthread_mutex_unlock(&mu);
        if (i >= round_n) return NULL;
        const uint64_t start = splitmix(seed * 0x100000001B3ull + round_base + i) & mask;
        uint64_t x = start, len = 0;
        do { x = f(x); ++len; } while ((x & dmask) && len < max_len);
        round_out[i] = (Trail){start, x, (x & dmask) ? 0 : len};
    }
}

// The two trails end on one point: step the longer one until both are as far from it, then both until they meet.
static int locate(Trail a, Trail b, uint64_t* xa, uint64_t* xb) {
    uint64_t pa = a.start, pb = b.start;
    for (; a.len > b.len; --a.len) pa = f(pa);
    for (; b.len > a.len; --b.len) pb = f(pb);
    if (pa == pb) return 0;                                       // one start lies on the other trail
    for (;;) {
        const uint64_t na = f(pa), nb = f(pb);
        if (na == nb) { *xa = pa; *xb = pb; return 1; }
        pa = na; pb = nb;
    }
}

static void print_pair(uint64_t a, uint64_t b) {
    if (mode == M_SIG) {
        if (extra && (a & 1)) { uint64_t t = a; a = b; b = t; }       // the longer allele second
        char sa[128], sb[128];
        const int na = allele_of(a, sa), nb = allele_of(b, sb);
        printf("sig%d %s %s 0x%016llx\n", sig_bits == 60 ? 4 : 8, sa, sb, (unsigned long long)make_sig(sa, na));
        if (make_sig(sa, na) != make_sig(sb, nb)) { fprintf(stderr, "internal error: no collision\n"); exit(1); }
        return;
    }
    if (mode == M_CLAW && !(a & 1)) { uint64_t t = a; a = b; b = t; }  // the QNAME (odd branch) first
    char sa[16], sb[16];
    name_of(a, sa);
    name_of(b, sb);
    const uint64_t ha = fnv_from(prefix_state, sa), hb = fnv_from(prefix_state, sb);
    printf("%s %s%s %s%s 0x%016llx\n", mode == M_CLAW ? "claw" : "name", prefix, sa, prefix, sb, (unsigned long long)ha);
    if (mode == M_NAME ? ha != hb : ha != (hb ^ REF_DOMAIN)) { fprintf(stderr, "internal error: no collision\n"); exit(1); }
}

int main(int argc, char** argv) {
    int threads = (int)sysconf(_SC_NPROCESSORS_ONLN), a = 1;
    for (; a + 1 < argc && argv[a][0] == '-'; a += 2) {
        if (!strcmp(argv[a], "-s")) seed = strtoull(argv[a + 1], NULL, 0);
        else if (!strcmp(argv[a], "-t")) threads = atoi(argv[a + 1]);
        else break;
    }
    if (a >= argc) goto usage;
    if (!strcmp(argv[a], "name") || !strcmp(argv[a], "claw")) {
        mode = strcmp(argv[a], "name") ? M_CLAW : M_NAME;
        if (a + 1 < argc) {
            if (strlen(argv[a + 1]) >= sizeof prefix) goto usage;
            strcpy(prefix, argv[a + 1]);
        }
        prefix_state = fnv_from(FNV_BASIS, prefix);
        bits = 64;
    } else if (!strcmp(argv[a], "sig") && a + 2 < argc) {
        mode = M_SIG;
        sig_bits = atoi(argv[a + 1]) == 4 ? 60 : atoi(argv[a + 1]) == 8 ? 56 : 0;
        anchor = argv[a + 2][0];
        if (!sig_bits || !strchr("ACGT", anchor) || argv[a + 2][1]) goto usage;
        extra = a + 3 < argc ? atoi(argv[a + 3]) : 0;
        if (extra < 0 || extra > 32) goto usage;
        bits = sig_bits;
    } else {
        goto usage;
    }
    if (threads < 1) threads = 1;
    mask = bits == 64 ? ~0ull : (1ull << bits) - 1;
    dbits = bits / 2 - 10;
    max_len = 20ull << dbits;
    const uint64_t per_round = (uint64_t)threads * 4;
    round_out = malloc(per_round * sizeof(Trail));
    uint64_t cap = 1 << 16, n_kept = 0;
    Trail* table = calloc(cap, sizeof(Trail));          // open addressing on dp; len == 0 marks an empty slot
    pthread_t* th = malloc((size_t)threads * sizeof(pthread_t));
    for (round_base = 0;; round_base += per_round) {
        round_n = per_round;
        next_trail = 0;
        for (int t = 0; t < threads; ++t) pthread_create(&th[t], NULL, worker, NULL);
        for (int t = 0; t < threads; ++t) pthread_join(th[t], NULL);
        for (uint64_t i = 0; i < round_n; ++i) {
            const Trail tr = round_out[i];
            if (!tr.len) continue;                                    // a trail caught in a cycle without a distinguished point
            uint64_t sl = splitmix(tr.dp) & (cap - 1);
            while (table[sl].len && table[sl].dp != tr.dp) sl = (sl + 1) & (cap - 1);
            if (table[sl].len) {
                uint64_t xa, xb;
                if (locate(table[sl], tr, &xa, &xb) && useful(xa, xb)) {
                    print_pair(xa, xb);
                    return 0;
                }
                continue;
            }
            table[sl] = tr;
            if (++n_kept * 2 > cap) { fprintf(stderr, "table full\n"); return 1; }
        }
    }
usage:
    fprintf(stderr, "usage: fnv_collide [-s SEED] [-t THREADS] name [PREFIX] | claw [PREFIX] | sig 4|8 A|C|G|T [EXTRA]\n");
    return 2;
}
