/*
 * dte_oracle.c — CPU ORACLE (test infrastructure only; see dte_oracle.h for the rules and the
 * "parity unpinned" statement).  Plain C11, no dependencies.  Build: see oracle/Makefile
 * (-O3 -fno-fast-math -ffp-contract=off so host float adds are single IEEE RNE operations).
 *
 * Every function cites the reference lines it restates (paths relative to the reference repository root).
 */
#define _GNU_SOURCE
#include "dte_oracle.h"
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <unistd.h>

/* ------------------------------------------------------------------------------------------ */
/* fp32 adder, model A: host float.                                                            */
/* FPAdder_2cycles_latency.v:360-369 rounds to nearest even; :376-386 has no subnormal results  */
/* (exponent underflow -> exception code 00 = zero) and FPAddersReduceTree.sv:141 /             */
/* FPAggregator.v:107-112 turn every "zero" result into the all-zero word (+0).                 */
/* Model A is exactly what the GPU executes with add.rn.ftz.f32: subnormal operands read as     */
/* signed zero, IEEE RNE add, subnormal results flushed to signed zero.  It coincides with the  */
/* netlist (model B below) on the contract domain: operands are +0 or normal finite, the result */
/* is exactly zero or normal finite.  tests/test_oracle_selfcheck.py diffs A against B.         */
/* ------------------------------------------------------------------------------------------ */
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

static inline uint32_t daz(uint32_t a) { return ((a & 0x7F800000u) == 0) ? (a & 0x80000000u) : a; }

uint32_t dteo_fpadd(uint32_t a, uint32_t b) {
    volatile float fa = u2f(daz(a)), fb = u2f(daz(b));
    volatile float fr = fa + fb;              /* one IEEE-754 binary32 RNE addition (SSE) */
    return daz(f2u(fr));
}

/* ------------------------------------------------------------------------------------------ */
/* fp32 adder, model B: bit-level restatement of the FloPoCo (wE=8, wF=23) single-path adder    */
/* datapath, FPAdder_2cycles_latency.v:296-387.  Numbers travel as 34-bit words                 */
/* {exc[1:0], sign, exp[7:0], frac[22:0]} with exc 00 = zero, 01 = normal, 10 = inf, 11 = NaN.  */
/* ------------------------------------------------------------------------------------------ */
typedef uint64_t fp34;

/* input wrapper {1'b0, |word, word}: FPAddersReduceTree.sv:94-95, FPAggregator.v:118 */
static inline fp34 fp34_wrap(uint32_t w) { return ((uint64_t)(w != 0) << 32) | w; }
/* output wrapper (exc == 00) ? 0 : word: FPAddersReduceTree.sv:141, FPAggregator.v:107-112 */
static inline uint32_t fp34_unwrap(fp34 r) { return ((r >> 32) & 3) == 0 ? 0u : (uint32_t)r; }

static fp34 fpadd34(fp34 X, fp34 Y) {
    /* :296-306 swap so that |newX| >= |newY| judged on {exc, exp, frac} */
    uint64_t keyX = ((X >> 32) & 3) << 31 | (X & 0x7FFFFFFFu);
    uint64_t keyY = ((Y >> 32) & 3) << 31 | (Y & 0x7FFFFFFFu);
    fp34 nX = keyX >= keyY ? X : Y, nY = keyX >= keyY ? Y : X;
    unsigned excX = (nX >> 32) & 3, excY = (nY >> 32) & 3;
    unsigned sX = (nX >> 31) & 1, sY = (nY >> 31) & 1;
    unsigned expX = (nX >> 23) & 0xFF, expY = (nY >> 23) & 0xFF;
    unsigned effSub = sX ^ sY;

    /* :313-320 exception class of the result before rounding */
    unsigned excRt;
    if (excX == 0 && excY == 0) excRt = 0;
    else if (excX <= 1 && excY <= 1) excRt = 1;                     /* at least one normal, no inf/NaN */
    else if (excX == 3 || excY == 3) excRt = 3;
    else if (excX == 2 && excY == 2) excRt = effSub ? 3 : 2;        /* inf-inf = NaN */
    else excRt = 2;
    /* :322 sign: (+0) + (-0) in either order is +0, otherwise the sign of the larger operand */
    unsigned signR = (excX == 0 && excY == 0 && (sX ^ sY)) ? 0 : sX;

    /* :324-330 align the smaller significand: 24-bit {1,frac} (0 if that operand is zero),
       26 guard positions, shift distance saturates at 26 */
    unsigned expDiff = (expX - expY) & 0x1FF;
    unsigned shiftVal = expDiff >= 25 ? 26 : (expDiff & 31);
    uint64_t fracY = excY == 0 ? 0 : (0x800000u | (nY & 0x7FFFFFu));
    uint64_t shifted = (fracY << 26) >> shiftVal;                   /* 50 bits */
    unsigned sticky = (shifted & 0xFFFFFFu) != 0;                   /* :333 */
    uint64_t fracYfar = (shifted >> 24) & 0x3FFFFFFu;               /* :336 27 bits, msb 0 */
    if (effSub) fracYfar ^= 0x7FFFFFFu;                             /* :337 */
    uint64_t fracXfar = (1ull << 25) | ((nX & 0x7FFFFFu) << 2);     /* :338 {01, frac, 00} */
    unsigned cin = effSub & !sticky;                                /* :339 */
    uint64_t sum = (fracXfar + fracYfar + cin) & 0x7FFFFFFu;        /* :340-344 27-bit adder */
    uint64_t grs = (sum << 1) | sticky;                             /* :346 28 bits */

    /* :348-353 / LZCShifter :133-146 leading-zero count by 16/8/4/2/1 with left shift */
    unsigned nz = 0; uint64_t v = grs & 0xFFFFFFFu;
    if ((v >> 12) == 0)          { nz |= 16; v = (v << 16) & 0xFFFFFFFu; }
    if ((v >> 20) == 0)          { nz |= 8;  v = (v << 8)  & 0xFFFFFFFu; }
    if ((v >> 24) == 0)          { nz |= 4;  v = (v << 4)  & 0xFFFFFFFu; }
    if ((v >> 26) == 0)          { nz |= 2;  v = (v << 2)  & 0xFFFFFFFu; }
    if ((v >> 27) == 0)          { nz |= 1;  v = (v << 1)  & 0xFFFFFFFu; }

    /* :356-369 exponent update and round to nearest even */
    uint64_t updExp = ((uint64_t)expX + 1 - nz) & 0x3FF;            /* 10 bits */
    unsigned eqdiffsign = nz == 31;
    uint64_t expFrac = (updExp << 24) | ((v >> 3) & 0xFFFFFFu);     /* 34 bits */
    unsigned stk = (v & 3) != 0, rnd = (v >> 2) & 1, grd = (v >> 3) & 1, lsb = (v >> 4) & 1;
    unsigned addRound = !(lsb == 0 && grd == 1 && rnd == 0 && stk == 0);
    uint64_t rounded = (expFrac + addRound) & 0x3FFFFFFFFull;
    unsigned upExc = (rounded >> 32) & 3;
    uint32_t fracR = (rounded >> 1) & 0x7FFFFFu, expR = (rounded >> 24) & 0xFF;

    /* :376-386 final exception code */
    unsigned excR2;
    if (excRt == 0) excR2 = 0;
    else if (excRt == 1) excR2 = upExc == 0 ? 1 : (upExc == 1 ? 2 : 0);   /* 01: overflow->inf, 1x: underflow->zero */
    else if (excRt == 2) excR2 = upExc <= 1 ? 2 : 3;
    else excR2 = 3;
    unsigned excR = (eqdiffsign && effSub) ? 0 : excR2;
    return ((uint64_t)excR << 32) | ((uint64_t)signR << 31) | ((uint64_t)expR << 23) | fracR;
}

uint32_t dteo_fpadd_literal(uint32_t a, uint32_t b) { return fp34_unwrap(fpadd34(fp34_wrap(a), fp34_wrap(b))); }

/* ------------------------------------------------------------------------------------------ */
/* Node step and walk, "clean" restatement on one tree given as heap arrays.                    */
/* DTPU.sv:594-596,710-712 children of n are 2n+1 / 2n+2; :628 feature index = FI[10:0];         */
/* :653 missing = raw equality; :655 signed compare of the raw words; :657-667 direction;        */
/* :588,663-665 exactly D iterations; :710,731 the leaf is the weight word of the child.         */
/* Bits 14 ("next node is leaf", :661) must be 0 here — complete trees only (SURVEY R3).         */
/* ------------------------------------------------------------------------------------------ */
uint32_t dteo_leaf(const dteo_cfg* c, const uint32_t* w, const uint16_t* fi, const uint32_t* x) {
    uint32_t n = 0;
    for (uint32_t lvl = 0; lvl < c->num_levels; ++lvl) {
        uint16_t f = fi[n];
        uint32_t v = x[f & 0x7FFu];
        uint32_t thr = w[n];
        int missing = (v == c->missing_value);
        int smaller = ((int32_t)v < (int32_t)thr);
        int right = missing ? ((f >> 13) & 1) : !smaller;
        n = 2 * n + 1 + (uint32_t)right;
        /* bit 14 "next node is leaf" (DTPU.sv:596,661,712): the children of this node are leaves, the walk ends in
           the child's cell.  BUILD-DEFINED where the RTL is broken: the RTL freezes node_offset without the
           direction bit while its read address keeps advancing, so with levels left it returns a wrong cell; the
           address-literal walker below keeps that behaviour, this one implements the evident intent (SURVEY R3). */
        if (f & 0x4000u) break;
    }
    return w[n];
}

/* reachable internal nodes must index inside the tuple; nodes below an early leaf are don't-care */
static int check_tree(const dteo_cfg* c, const uint16_t* fi, size_t F) {
    const uint32_t n_int = (1u << c->num_levels) - 1;
    uint8_t* dead = (uint8_t*)calloc(n_int ? n_int : 1, 1);
    if (!dead) return -5;
    int rc = 0;
    for (uint32_t i = 0; i < n_int && !rc; ++i) {
        if ((dead[i] || (fi[i] & 0x4000u)) && 2 * i + 2 < n_int) dead[2 * i + 1] = dead[2 * i + 2] = 1;
        if (!dead[i] && (fi[i] & 0x7FFu) >= F) rc = -3;
    }
    free(dead);
    return rc;
}

/* 8-leaf reduce tree ((l0+l1)+(l2+l3))+((l4+l5)+(l6+l7)): FPAddersReduceTree.sv:90-125, output
   wrapper :141.  Model A version on 32-bit words. */
static inline uint32_t tree8_a(const uint32_t* l) {
    uint32_t a = dteo_fpadd(l[0], l[1]), b = dteo_fpadd(l[2], l[3]);
    uint32_t cc = dteo_fpadd(l[4], l[5]), d = dteo_fpadd(l[6], l[7]);
    return dteo_fpadd(dteo_fpadd(a, b), dteo_fpadd(cc, d));
}
/* Model B version: 34-bit words flow between the adder levels without re-wrapping. */
static inline uint32_t tree8_b(const uint32_t* l) {
    fp34 a = fpadd34(fp34_wrap(l[0]), fp34_wrap(l[1])), b = fpadd34(fp34_wrap(l[2]), fp34_wrap(l[3]));
    fp34 cc = fpadd34(fp34_wrap(l[4]), fp34_wrap(l[5])), d = fpadd34(fp34_wrap(l[6]), fp34_wrap(l[7]));
    return fp34_unwrap(fpadd34(fpadd34(a, b), fpadd34(cc, d)));
}

static int check_cfg(const dteo_cfg* c) {
    if (c->num_levels < 1 || c->num_levels > 15) return -1;
    if (c->clusters < 1 || c->clusters > 8) return -1;
    if (c->trees_per_pu < 1) return -1;
    if (c->tuple_cls < 1) return -1;
    if ((uint64_t)c->tree_w_cls * 4 < (2ull << c->num_levels) - 1) return -1;   /* 2^(D+1)-1 words */
    if ((uint64_t)c->tree_f_cls * 8 < (1ull << c->num_levels) - 1) return -1;   /* 2^D-1 indexes   */
    return 0;
}

/* One tuple, placement and summation order:
 *   tree t (arrival order) -> PU t%8, cluster (t/8)%K, slot t/(8K)   Core.sv:291-304,352-367
 *   per cluster: for slot s: r = tree8(leaves of the 8 PUs); acc = r + acc   FPAddersReduceTree.sv,
 *                FPAggregator.v:79-131 (acc starts at 0, "X = input, Y = prev")
 *   slots beyond S are never issued (DTPU.sv:519-531); slots without a programmed tree give 0
 *                (DTPU.sv:544,760)
 *   across clusters: acc = part_c + acc for c = 0..K-1   Core.sv:486-542
 */
static uint32_t score_one(const dteo_cfg* c, const uint32_t* W, const uint16_t* FI,
                          const uint32_t* x, int literal_adder) {
    const uint32_t K = c->clusters, S = c->trees_per_pu, T = c->num_trees;
    const size_t wstride = (size_t)c->tree_w_cls * 4, fstride = (size_t)c->tree_f_cls * 8;
    fp34 tot_b = 0; uint32_t tot_a = 0;
    for (uint32_t j = 0; j < K; ++j) {
        fp34 acc_b = 0; uint32_t acc_a = 0;
        for (uint32_t s = 0; s < S; ++s) {
            uint64_t g = (uint64_t)s * K + j;
            uint32_t l[8];
            for (uint32_t p = 0; p < 8; ++p) {
                uint64_t t = g * 8 + p;
                l[p] = t < T ? dteo_leaf(c, W + t * wstride, FI + t * fstride, x) : 0u;
            }
            if (literal_adder) acc_b = fpadd34(fp34_wrap(tree8_b(l)), acc_b);
            else acc_a = dteo_fpadd(tree8_a(l), acc_a);
        }
        if (literal_adder) tot_b = fpadd34(fp34_wrap(fp34_unwrap(acc_b)), tot_b);
        else tot_a = dteo_fpadd(acc_a, tot_a);
    }
    return literal_adder ? fp34_unwrap(tot_b) : tot_a;
}

int dteo_online_cpus(void) {
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    return n > 0 ? (int)n : 1;
}

/* CPUs this process may actually use: online CPUs, cut by the affinity mask, cut by the cgroup CPU quota
   (cgroup v2 cpu.max "quota period", v1 cpu.cfs_quota_us / cpu.cfs_period_us).  The quota matters: a 1-GPU
   lease on a 128-thread host can be capped at ~11 cores, and 128 busy threads then only thrash. */
int dteo_max_threads(void) {
    long n = dteo_online_cpus();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) {
        int c = CPU_COUNT(&set);
        if (c > 0 && c < n) n = c;
    }
    double quota = -1, period = -1;
    FILE* fh = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (fh) {
        char q[64];
        if (fscanf(fh, "%63s %lf", q, &period) == 2 && q[0] != 'm') quota = atof(q);
        fclose(fh);
    } else {
        FILE* fq = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r");
        FILE* fp = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
        if (fq && fp && fscanf(fq, "%lf", &quota) == 1 && fscanf(fp, "%lf", &period) == 1) { /* both read */ }
        if (fq) fclose(fq);
        if (fp) fclose(fp);
    }
    if (quota > 0 && period > 0) {
        long c = (long)((quota + period - 1) / period);
        if (c < 1) c = 1;
        if (c < n) n = c;
    }
    return n > 0 ? (int)n : 1;
}

typedef struct {
    const dteo_cfg* c; const uint32_t* W; const uint16_t* FI; const uint32_t* X;
    uint32_t* scores; size_t lo, hi, F; int literal_adder;
} score_job;

static void* score_worker(void* arg) {
    score_job* j = (score_job*)arg;
    for (size_t i = j->lo; i < j->hi; ++i)
        j->scores[i] = score_one(j->c, j->W, j->FI, j->X + i * j->F, j->literal_adder);
    return NULL;
}

int dteo_scores(const dteo_cfg* c, const void* weights_cls, const void* findex_cls,
                const void* tuple_cls, size_t n, uint32_t* scores, int literal_adder, int threads) {
    if (check_cfg(c)) return -1;
    const uint32_t* W = (const uint32_t*)weights_cls;
    const uint16_t* FI = (const uint16_t*)findex_cls;
    const uint32_t* X = (const uint32_t*)tuple_cls;
    const size_t F = (size_t)c->tuple_cls * 4;
    /* out-of-contract inputs are refused, not guessed: a reachable feature index beyond the tuple */
    for (uint32_t t = 0; t < c->num_trees; ++t) {
        int rc = check_tree(c, FI + (size_t)t * c->tree_f_cls * 8, F);
        if (rc) return rc;
    }
    if (threads < 1) threads = 1;
    if ((size_t)threads > n) threads = n ? (int)n : 1;
    if (threads == 1) {
        score_job j = {c, W, FI, X, scores, 0, n, F, literal_adder};
        score_worker(&j);
        return 0;
    }
    /* tuples are independent: static contiguous split over plain pthreads */
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
    score_job* jobs = (score_job*)malloc(sizeof(score_job) * (size_t)threads);
    if (!th || !jobs) { free(th); free(jobs); return -5; }
    for (int k = 0; k < threads; ++k) {
        size_t lo = n * (size_t)k / (size_t)threads, hi = n * (size_t)(k + 1) / (size_t)threads;
        score_job j = {c, W, FI, X, scores, lo, hi, F, literal_adder};
        jobs[k] = j;
        if (pthread_create(&th[k], NULL, score_worker, &jobs[k])) { score_worker(&jobs[k]); th[k] = 0; }
    }
    for (int k = 0; k < threads; ++k) if (th[k]) pthread_join(th[k], NULL);
    free(th); free(jobs);
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Tree-blocked evaluation order — the SAME arithmetic as score_one() (model-A adder), the same   */
/* per-tuple summation order, but the loops are interchanged so that one tree8 group is walked by */
/* a block of tuples before the next group is touched: the 8 trees (8 x 10*2^D bytes) stay in     */
/* cache instead of the whole ensemble streaming past every tuple.  For a fixed tuple the         */
/* operation sequence is unchanged: per cluster j, slots s ascending: acc_j = tree8(...) + acc_j  */
/* (FPAggregator.v:79-131); then tot = acc_j + tot, j ascending (Core.sv:486-542).  This is the   */
/* loop timed as the CPU baseline; tests assert it is bit-identical to dteo_scores().             */
/* ------------------------------------------------------------------------------------------ */
#define DTEO_BLOCK 64
static void score_block(const dteo_cfg* c, const uint32_t* W, const uint16_t* FI, const uint32_t* X, size_t F,
                        size_t nb, uint32_t* out) {
    const uint32_t K = c->clusters, S = c->trees_per_pu, T = c->num_trees;
    const size_t wstride = (size_t)c->tree_w_cls * 4, fstride = (size_t)c->tree_f_cls * 8;
    uint32_t acc[DTEO_BLOCK][8];
    uint32_t leaf[DTEO_BLOCK][8];
    memset(acc, 0, sizeof acc);
    for (uint32_t s = 0; s < S; ++s) {
        for (uint32_t j = 0; j < K; ++j) {
            const uint64_t g = (uint64_t)s * K + j;
            for (uint32_t p = 0; p < 8; ++p) {
                const uint64_t t = g * 8 + p;
                if (t < T) {
                    const uint32_t* w = W + t * wstride;
                    const uint16_t* fi = FI + t * fstride;
                    for (size_t b = 0; b < nb; ++b) leaf[b][p] = dteo_leaf(c, w, fi, X + b * F);
                } else {
                    for (size_t b = 0; b < nb; ++b) leaf[b][p] = 0u;
                }
            }
            for (size_t b = 0; b < nb; ++b) acc[b][j] = dteo_fpadd(tree8_a(leaf[b]), acc[b][j]);
        }
    }
    for (size_t b = 0; b < nb; ++b) {
        uint32_t tot = 0;
        for (uint32_t j = 0; j < K; ++j) tot = dteo_fpadd(acc[b][j], tot);
        out[b] = tot;
    }
}

static void* blocked_worker(void* arg) {
    score_job* j = (score_job*)arg;
    for (size_t i = j->lo; i < j->hi; i += DTEO_BLOCK) {
        size_t nb = j->hi - i < DTEO_BLOCK ? j->hi - i : DTEO_BLOCK;
        score_block(j->c, j->W, j->FI, j->X + i * j->F, j->F, nb, j->scores + i);
    }
    return NULL;
}

int dteo_scores_blocked(const dteo_cfg* c, const void* weights_cls, const void* findex_cls,
                        const void* tuple_cls, size_t n, uint32_t* scores, int threads) {
    if (check_cfg(c)) return -1;
    const uint32_t* W = (const uint32_t*)weights_cls;
    const uint16_t* FI = (const uint16_t*)findex_cls;
    const uint32_t* X = (const uint32_t*)tuple_cls;
    const size_t F = (size_t)c->tuple_cls * 4;
    for (uint32_t t = 0; t < c->num_trees; ++t) {
        int rc = check_tree(c, FI + (size_t)t * c->tree_f_cls * 8, F);
        if (rc) return rc;
    }
    if (threads < 1) threads = 1;
    size_t nblocks = (n + DTEO_BLOCK - 1) / DTEO_BLOCK;
    if ((size_t)threads > nblocks) threads = nblocks ? (int)nblocks : 1;
    if (threads == 1) {
        score_job j = {c, W, FI, X, scores, 0, n, F, 0};
        blocked_worker(&j);
        return 0;
    }
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
    score_job* jobs = (score_job*)malloc(sizeof(score_job) * (size_t)threads);
    if (!th || !jobs) { free(th); free(jobs); return -5; }
    for (int k = 0; k < threads; ++k) {              /* whole blocks per thread, contiguous */
        size_t lo = nblocks * (size_t)k / (size_t)threads * DTEO_BLOCK, hi = nblocks * (size_t)(k + 1) / (size_t)threads * DTEO_BLOCK;
        if (hi > n) hi = n;
        score_job j = {c, W, FI, X, scores, lo, hi, F, 0};
        jobs[k] = j;
        if (pthread_create(&th[k], NULL, blocked_worker, &jobs[k])) { blocked_worker(&jobs[k]); th[k] = 0; }
    }
    for (int k = 0; k < threads; ++k) if (th[k]) pthread_join(th[k], NULL);
    free(th); free(jobs);
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Address-literal restatement: the PU memories as the hardware fills them, walked with the     */
/* hardware's address arithmetic and field widths.  Independent of dteo_leaf/score_one above.   */
/*   WeightsMem 2048 lines x 4 words (DTPU.sv:282-301, write pointer :307-319)                   */
/*   TreeFeatureIndex_Mem 1024 lines x 8 halfwords (:322-338, write pointer :347-354)            */
/*   SamplesFeatures_Mem 512 lines x 4 words, circular (:360-399)                                */
/*   per-slot tree offsets accumulate by lines-per-tree (:512-531) — the TRUE line counts        */
/*   (the RTL wires the minus-one CSR copies there, DTInference.sv:505-506; SURVEY R10 fixes it) */
/*   walk registers and widths :579-596,690-720; leaf read :731-761.                             */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
    uint32_t w[2048][4];
    uint16_t f[1024][8];
    uint32_t x[512][4];
    uint32_t w_wr, f_wr, ntrees;
} pu_mem;

static uint32_t pu_walk(const pu_mem* m, const dteo_cfg* c, uint32_t slot, uint32_t tuple_off) {
    if (slot >= m->ntrees) return 0;                                   /* instr_NOP -> EMPTY -> leaf 0 */
    const uint32_t w_off = (slot * c->tree_w_cls) & 0x7FF;             /* 11-bit line offsets */
    const uint32_t f_off = (slot * c->tree_f_cls) & 0x7FF;
    uint32_t w_addr = (w_off << 2) & 0x1FFF;                           /* 13-bit word address */
    uint32_t f_addr = ((f_off & 0x3FF) << 3) & 0x1FFF;
    uint32_t node_off = 0, nop = 0;
    for (uint32_t level = 0;; ++level) {
        uint32_t thr = m->w[w_addr >> 2][w_addr & 3];
        uint16_t fi = m->f[f_addr >> 3][f_addr & 7];
        uint32_t next_w = ((w_off << 2) + (((node_off & 0xFFF) << 1) | 1)) & 0x1FFF;
        uint32_t next_f = (((f_off & 0x3FF) << 3) + (((node_off & 0xFFF) << 1) | 1)) & 0x1FFF;
        uint32_t next_off = nop ? node_off : ((((node_off & 0xFFF) << 1) | 1) & 0x1FFF);
        uint32_t x_addr = ((fi & 0x7FFu) + (tuple_off << 2)) & 0x7FF;  /* 11-bit word address */
        uint32_t v = m->x[x_addr >> 2][x_addr & 3];
        uint32_t missing = v == c->missing_value;
        /* 33-bit unsigned compare with the inverted sign bit prepended (:655) */
        uint64_t a = ((uint64_t)(~v >> 31) << 32) | v, b = ((uint64_t)(~thr >> 31) << 32) | thr;
        uint32_t incr = missing ? ((fi >> 13) & 1) : !(a < b);
        uint32_t nop_next = nop | ((fi >> 14) & 1);
        w_addr = (next_w + incr) & 0x1FFF;
        f_addr = (next_f + incr) & 0x1FFF;
        node_off = nop_next ? next_off : ((next_off + incr) & 0x1FFF);
        nop = nop_next;
        if (level == c->num_levels - 1) break;                         /* isLastLevel (:663) */
    }
    return m->w[w_addr >> 2][w_addr & 3];                              /* port-B leaf read */
}

int dteo_scores_literal(const dteo_cfg* c, const void* weights_cls, const void* findex_cls,
                        const void* tuple_cls, size_t n, uint32_t* scores) {
    if (check_cfg(c)) return -1;
    const uint32_t K = c->clusters, S = c->trees_per_pu;
    if (!(K == 1 || K == 2 || K == 4 || K == 8)) return -2;            /* rotating schedules, RLS.v:35-58 */
    if (c->num_levels > 12 || S > 16) return -2;
    if ((uint64_t)S * c->tree_w_cls > 2048 || (uint64_t)S * c->tree_f_cls > 1024) return -2;
    if (c->tuple_cls > 512) return -2;
    pu_mem* pus = (pu_mem*)calloc((size_t)K * 8, sizeof(pu_mem));
    if (!pus) return -5;
    const uint32_t(*WL)[4] = (const uint32_t(*)[4])weights_cls;
    const uint16_t(*FL)[8] = (const uint16_t(*)[8])findex_cls;
    const uint32_t(*XL)[4] = (const uint32_t(*)[4])tuple_cls;
    int rc = 0;
    /* PROG: weights stream first, then index stream, each restarting the schedule
       (Core.sv:291-304); tree t -> PU t%8 (:352-367), cluster (t/8)%K of every replica group */
    for (uint32_t t = 0; t < c->num_trees && !rc; ++t) {
        pu_mem* m = &pus[((t / 8) % K) * 8 + (t % 8)];
        if (m->w_wr + c->tree_w_cls > 2048 || m->f_wr + c->tree_f_cls > 1024) { rc = -2; break; }
        for (uint32_t i = 0; i < c->tree_w_cls; ++i) memcpy(m->w[m->w_wr++], WL[(size_t)t * c->tree_w_cls + i], 16);
        for (uint32_t i = 0; i < c->tree_f_cls; ++i) memcpy(m->f[m->f_wr++], FL[(size_t)t * c->tree_f_cls + i], 16);
        m->ntrees++;
    }
    uint32_t x_wr = 0;                                                 /* features_wr_addr, 9 bits */
    for (size_t i = 0; i < n && !rc; ++i) {
        uint32_t tuple_off = x_wr;
        for (uint32_t l = 0; l < c->tuple_cls; ++l) {
            for (uint32_t q = 0; q < K * 8; ++q) memcpy(pus[q].x[x_wr], XL[i * c->tuple_cls + l], 16);
            x_wr = (x_wr + 1) & 0x1FF;
        }
        fp34 tot = 0;
        for (uint32_t j = 0; j < K; ++j) {
            fp34 acc = 0;
            for (uint32_t s = 0; s < S; ++s) {
                uint32_t l8[8];
                for (uint32_t p = 0; p < 8; ++p) l8[p] = pu_walk(&pus[j * 8 + p], c, s, tuple_off);
                acc = fpadd34(fp34_wrap(tree8_b(l8)), acc);
            }
            tot = fpadd34(fp34_wrap(fp34_unwrap(acc)), tot);
        }
        scores[i] = fp34_unwrap(tot);
    }
    free(pus);
    return rc;
}

/* ResultsCombiner aggregate mode: the host node injects its local line, every following node
   emits local + incoming, lane-wise (ResultsCombiner.sv:292-311,359-368).  The adders there are
   fed {1'b0, |word, word} just like the in-core ones. */
void dteo_ring_combine(const uint32_t* const* partials, int G, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) {
        uint32_t acc = partials[0][i];
        for (int g = 1; g < G; ++g) acc = dteo_fpadd(partials[g][i], acc);
        out[i] = acc;
    }
}

/* ResultsCombiner line packing (ResultsCombiner.sv:132-162): local results fill words curr_word = 0..3 of a
   128-bit line; the line is emitted when the 4th word is written; fewer than 4 trailing results never leave. */
size_t dteo_result_lines(const uint32_t* scores, size_t n, uint32_t* lines) {
    uint32_t line[4] = {0, 0, 0, 0};
    unsigned curr_word = 0;
    size_t out = 0;
    for (size_t i = 0; i < n; ++i) {
        line[curr_word] = scores[i];
        if (curr_word == 3) { memcpy(lines + 4 * out, line, 16); ++out; }
        curr_word = (curr_word + 1) & 3;
    }
    return out;
}

void dteo_labels(const uint32_t* scores, size_t n, uint8_t* labels) {
    for (size_t i = 0; i < n; ++i) labels[i] = u2f(scores[i]) > 0.0f ? 1 : 0;
}
