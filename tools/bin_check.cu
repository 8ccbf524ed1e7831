// bin_check.cu — HOST-ONLY check of the binned layout (bin_edges and pack_ensemble's binned records in dte_device.cuh):
// builds the edge table over every tree of the streams, packs trees [first, first + T) with it, bins the fp32 tuples on
// the host, then decodes the 4-byte tops and the rank-coded bottom records exactly as the binned kernels do and prints
// the leaf word of every (tuple, tree).  tests/test_binned_layout.py compares them with the oracle's dteo_leaf on the
// fp32 tuples, so the exactness of the binned layout is covered by the CPU test tier.  Test infrastructure.
//   bin_check <D> <F> <T> <n> <missing> <weights.bin> <findex.bin> <tuples.bin> <classes> <first> <edges.bin>
//     ->  n*T uint32 leaf words (binary, stdout), tree t = stream tree first + t, in stream order;
//         edges.bin = offsets[F + 1] then the edges (uint32)
// Exit 6 (message on stderr) when bin_edges refuses the streams; 5 when a class-padding slot decodes to a leaf != +0.
#include "../distributed-decisiontrees_b200/csrc/dte_device.cuh"
#include <cstdio>
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

// bin_tuples_kernel on the host: #{edges <= x} in int32 order, 255 for the missing pattern
static uint8_t bin_of(const BinEdges& be, uint32_t f, uint32_t x, uint32_t missing) {
    if (x == missing) return 255;
    uint32_t b = 0;
    for (uint32_t j = be.offsets[f]; j < be.offsets[f + 1]; ++j) b += (int32_t)x >= (int32_t)be.edges[j];
    return (uint8_t)b;
}

// leaf word of tree slot `slot` of the binned layout for bins b, decoded as dt_walk_tile<..., BIN> decodes it
static uint32_t walk(const PackedEnsemble& pk, uint32_t slot, const uint8_t* b) {
    const EnsembleShape& sh = pk.shape;
    const int BV = sh.wide ? 4 : 2;
    const uint32_t missing = 255;
    // top: byte offset o into the tree's 4-byte records, child = 2o + 4 + 4*right
    uint32_t o = 0;
    const uint32_t* tp = pk.top_b.data() + (size_t)slot * sh.top_stride;
    for (uint32_t lvl = 0; lvl < sh.Dtop; ++lvl) {
        const uint32_t w = tp[o / 4];
        const uint32_t xv = b[(w >> 8) & 0x7FFu], thr = w & 0xFFu;
        const bool right = (xv == missing) ? (w >= (1u << 20)) : !((int32_t)xv < (int32_t)thr);
        o = 2 * o + (right ? 8u : 4u);
    }
    const uint32_t j = (o >> 2) - (sh.nb - 1);
    const uint4* rec = pk.bottom_b.data() + ((size_t)slot * sh.nb + j) * BV;
    uint32_t fp, fl_, fr, mp, ml, mr; uint4 leaves;
    if (sh.wide) {
        fp = rec[0].w & 0xFFFFu; mp = rec[0].w >> 16; fl_ = rec[1].x & 0xFFFFu; ml = rec[1].x >> 16;
        fr = rec[1].y & 0xFFFFu; mr = rec[1].y >> 16; leaves = rec[2];
    } else {
        const uint32_t k = rec[0].w;
        fp = k & 0x1FFu; mp = (k >> 9) & 1u; fl_ = (k >> 10) & 0x1FFu; ml = (k >> 19) & 1u; fr = (k >> 20) & 0x1FFu; mr = (k >> 29) & 1u;
        leaves = rec[1];
    }
    const uint32_t xp = b[fp];
    const bool r1 = (xp == missing) ? (mp != 0) : !((int32_t)xp < (int32_t)rec[0].x);
    const uint32_t thr = r1 ? rec[0].z : rec[0].y, xc = b[r1 ? fr : fl_], mc = r1 ? mr : ml;
    const bool r2 = (xc == missing) ? (mc != 0) : !((int32_t)xc < (int32_t)thr);
    return r1 ? (r2 ? leaves.w : leaves.z) : (r2 ? leaves.y : leaves.x);
}

int main(int argc, char** argv) {
    if (argc < 12) return 2;
    Geom g;
    g.D = (uint32_t)atoi(argv[1]); const uint32_t F = (uint32_t)atoi(argv[2]), T = (uint32_t)atoi(argv[3]);
    const size_t n = (size_t)atoll(argv[4]);
    g.missing = (uint32_t)strtoul(argv[5], nullptr, 0);
    g.K = 1; g.S = 1; g.tuple_cls = F / 4;
    g.w_cls = (uint32_t)(((2ull << g.D) - 1 + 3) / 4); g.f_cls = (uint32_t)(((1ull << g.D) - 1 + 7) / 8);
    auto wl = slurp(argv[6]), fl = slurp(argv[7]), xs = slurp(argv[8]);
    const uint32_t C = (uint32_t)atoi(argv[9]), first = (uint32_t)atoi(argv[10]);
    BinEdges be;
    std::string msg;
    int rc = bin_edges(g, wl.data(), wl.size() / 16, fl.data(), fl.size() / 16, be, msg);
    if (rc) { fprintf(stderr, "bin_edges: %d %s\n", rc, msg.c_str()); return 6; }
    FILE* ef = fopen(argv[11], "wb");
    if (!ef) return 2;
    fwrite(be.offsets.data(), 4, be.offsets.size(), ef);
    fwrite(be.edges.data(), 4, be.edges.size(), ef);
    fclose(ef);
    PackedEnsemble pk;
    rc = pack_ensemble(g, wl.data(), wl.size() / 16, fl.data(), fl.size() / 16, first, T, C, pk, msg, &be);
    if (rc) { fprintf(stderr, "pack_ensemble: %d %s\n", rc, msg.c_str()); return 3; }
    const EnsembleShape& sh = pk.shape;
    if (sh.T != T || sh.C != C || pk.top_b.size() != (size_t)sh.Tpad * sh.top_stride || pk.bottom_b.size() != pk.bottom.size()) return 4;
    // class-major slot of every stream tree, as tools/pack_check derives it
    std::vector<uint32_t> per(C, 0), slot(T);
    for (uint32_t t = 0; t < T; ++t) slot[t] = per[(first + t) % C]++;
    std::vector<uint8_t> used(sh.Tpad, 0);
    for (uint32_t t = 0; t < T; ++t) { slot[t] += ((first + t) % C) * sh.gpc * 8; used[slot[t]] = 1; }
    const uint32_t* X = reinterpret_cast<const uint32_t*>(xs.data());
    std::vector<uint32_t> out(n * T);
    std::vector<uint8_t> b(F);
    for (size_t i = 0; i < n; ++i) {
        for (uint32_t f = 0; f < F; ++f) b[f] = bin_of(be, f, X[i * F + f], g.missing);
        for (uint32_t t = 0; t < T; ++t) out[i * T + t] = walk(pk, slot[t], b.data());
        for (uint32_t s = 0; s < sh.Tpad; ++s)
            if (!used[s] && walk(pk, s, b.data()) != 0u) {
                fprintf(stderr, "padding slot %u gives a non-zero leaf for tuple %zu\n", s, i);
                return 5;
            }
    }
    fwrite(out.data(), 4, out.size(), stdout);
    return 0;
}
