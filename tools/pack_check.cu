// pack_check.cu — HOST-ONLY check of the ensemble repacker (pack_ensemble in dte_device.cuh): packs the reference
// streams into the device layout (8-byte top records + 32/64-byte bottom records, early leaves expanded), then decodes
// that layout on the CPU exactly as the kernels do and prints the leaf word of every (tuple, tree).  tests/ compare it
// with the oracle's dteo_leaf — so the repacker is covered by the CPU test tier (no GPU needed).  Test infrastructure.
//   pack_check <D> <F> <T> <n> <missing> <weights.bin> <findex.bin> <tuples.bin> [<classes> [<first>]]
//     ->  n*T uint32 leaf words (binary, stdout), tree t = stream tree first + t
// With <classes> the T trees starting at stream tree <first> are packed as a multi-class ensemble (class-major, every
// class padded to whole tree8 groups).  The class-major permutation is undone here from the stream index alone, so the
// leaves come out in stream order; every padding slot must decode to the leaf +0 for every tuple (exit 5 otherwise).
//   pack_check leaf <same arguments>
//     ->  n*T uint16 leaf cells (binary, stdout): the leaf-id layout (bottom_id) packed as well and decoded as the leaf
//         walks decode it, the cell in the stream tree's own heap that each (tuple, tree) ends in
#include "../distributed-decisiontrees_b200/csrc/dte_device.cuh"
#include <cstdio>
#include <cstring>
using namespace dte;

static std::vector<unsigned char> slurp(const char* p) {
    std::vector<unsigned char> v;
    FILE* f = fopen(p, "rb");
    if (!f) return v;
    fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
    v.resize((size_t)n);
    if (fread(v.data(), 1, (size_t)n, f) != (size_t)n) v.clear();
    fclose(f);
    return v;
}

// leaf word of tree slot `slot` of the packed layout for tuple x, decoded as the kernels decode it
// `bottom`: pk.bottom (leaf words) or pk.bottom_id (leaf cells)
static uint32_t walk(const PackedEnsemble& pk, uint32_t slot, const uint32_t* x, uint32_t missing, const std::vector<uint4>& bottom) {
    const EnsembleShape& sh = pk.shape;
    const int BV = sh.wide ? 4 : 2;
    // top: byte offset o into the tree's 8-byte heap records, child = 2o + 8 + 8*right  (step_inc in dte_kernels.cuh)
    uint32_t o = 0;
    const uint2* tp = pk.top.data() + (size_t)slot * sh.top_stride;
    for (uint32_t lvl = 0; lvl < sh.Dtop; ++lvl) {
        const uint2 nd = tp[o / 8];
        const uint32_t xv = x[nd.y & 0xFFFFu];
        uint32_t inc = ((int32_t)xv < (int32_t)nd.x) ? 8u : 16u;
        if (xv == missing) inc = nd.y >> 16;
        o = 2 * o + inc;
    }
    const uint32_t j = (o >> 3) - (sh.nb - 1);
    const uint4* rec = bottom.data() + ((size_t)slot * sh.nb + j) * BV;
    uint32_t fp, fl_, fr, mp, ml, mr; uint4 leaves;
    if (sh.wide) {
        fp = rec[0].w & 0xFFFFu; mp = rec[0].w >> 16; fl_ = rec[1].x & 0xFFFFu; ml = rec[1].x >> 16;
        fr = rec[1].y & 0xFFFFu; mr = rec[1].y >> 16; leaves = rec[2];
    } else {
        const uint32_t k = rec[0].w;
        fp = k & 0x1FFu; mp = (k >> 9) & 1u; fl_ = (k >> 10) & 0x1FFu; ml = (k >> 19) & 1u; fr = (k >> 20) & 0x1FFu; mr = (k >> 29) & 1u;
        leaves = rec[1];
    }
    const uint32_t xp = x[fp];
    const bool r1 = (xp == missing) ? (mp != 0) : !((int32_t)xp < (int32_t)rec[0].x);
    const uint32_t thr = r1 ? rec[0].z : rec[0].y, xc = x[r1 ? fr : fl_], mc = r1 ? mr : ml;
    const bool r2 = (xc == missing) ? (mc != 0) : !((int32_t)xc < (int32_t)thr);
    return r1 ? (r2 ? leaves.w : leaves.z) : (r2 ? leaves.y : leaves.x);
}

int main(int argc, char** argv) {
    const bool leaf = argc > 1 && !strcmp(argv[1], "leaf");
    if (leaf) { --argc; ++argv; }
    if (argc < 9) return 2;
    Geom g;
    g.D = (uint32_t)atoi(argv[1]); const uint32_t F = (uint32_t)atoi(argv[2]), T = (uint32_t)atoi(argv[3]);
    const size_t n = (size_t)atoll(argv[4]);
    g.missing = (uint32_t)strtoul(argv[5], nullptr, 0);
    g.K = 1; g.S = 1; g.tuple_cls = F / 4;
    g.w_cls = (uint32_t)(((2ull << g.D) - 1 + 3) / 4); g.f_cls = (uint32_t)(((1ull << g.D) - 1 + 7) / 8);
    auto wl = slurp(argv[6]), fl = slurp(argv[7]), xs = slurp(argv[8]);
    const bool classed = argc > 9;
    const uint32_t C = classed ? (uint32_t)atoi(argv[9]) : 1u, first = argc > 10 ? (uint32_t)atoi(argv[10]) : 0u;
    PackedEnsemble pk;
    std::string msg;
    int rc = classed ? pack_ensemble(g, wl.data(), wl.size() / 16, fl.data(), fl.size() / 16, first, T, C, pk, msg, nullptr, leaf)
                     : pack_ensemble(g, wl.data(), wl.size() / 16, fl.data(), fl.size() / 16, 0, 0, 1, pk, msg, nullptr, leaf);
    if (rc) { fprintf(stderr, "pack_ensemble: %d %s\n", rc, msg.c_str()); return 3; }
    const EnsembleShape& sh = pk.shape;
    if (sh.T != T || sh.C != C) return 4;
    // the class-major slot of every stream tree, derived independently of the packer: class c = (first + t) % C,
    // k-th tree of its class -> slot c * gpc * 8 + k, gpc = ceil(largest class / 8)
    std::vector<uint32_t> per(C, 0), slot(T);
    for (uint32_t t = 0; t < T; ++t) slot[t] = per[(first + t) % C]++;
    uint32_t cmax = 0;
    for (uint32_t c = 0; c < C; ++c) cmax = std::max(cmax, per[c]);
    const uint32_t gpc = (cmax + 7) / 8;
    if (sh.gpc != gpc || sh.cls_max != cmax || sh.Tpad != C * gpc * 8) {
        fprintf(stderr, "shape: gpc %u (want %u) cls_max %u (want %u) Tpad %u\n", sh.gpc, gpc, sh.cls_max, cmax, sh.Tpad);
        return 4;
    }
    std::vector<uint8_t> used(sh.Tpad, 0);
    for (uint32_t t = 0; t < T; ++t) { slot[t] += ((first + t) % C) * gpc * 8; used[slot[t]] = 1; }
    const uint32_t* X = reinterpret_cast<const uint32_t*>(xs.data());
    if (leaf) {
        if (pk.bottom_id.size() != pk.bottom.size()) return 4;
        std::vector<uint16_t> cells(n * T);
        for (size_t i = 0; i < n; ++i)
            for (uint32_t t = 0; t < T; ++t) {
                const uint32_t c = walk(pk, slot[t], X + i * F, g.missing, pk.bottom_id);
                if (c > 0xFFFFu) return 6;
                cells[i * T + t] = (uint16_t)c;
            }
        fwrite(cells.data(), 2, cells.size(), stdout);
        return 0;
    }
    std::vector<uint32_t> out(n * T);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t* x = X + i * F;
        for (uint32_t t = 0; t < T; ++t) out[i * T + t] = walk(pk, slot[t], x, g.missing, pk.bottom);
        for (uint32_t s = 0; s < sh.Tpad; ++s)
            if (!used[s] && walk(pk, s, x, g.missing, pk.bottom) != 0u) {
                fprintf(stderr, "padding slot %u gives a non-zero leaf for tuple %zu\n", s, i);
                return 5;
            }
    }
    fwrite(out.data(), 4, out.size(), stdout);
    return 0;
}
