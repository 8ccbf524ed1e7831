// pack_check.cu — HOST-ONLY check of the ensemble repacker (pack_ensemble in dte_device.cuh): packs the reference
// streams into the device layout (8-byte top records + 32/64-byte bottom records, early leaves expanded), then decodes
// that layout on the CPU exactly as the kernels do and prints the leaf word of every (tuple, tree).  tests/ compare it
// with the oracle's dteo_leaf — so the repacker is covered by the CPU test tier (no GPU needed).  Test infrastructure.
//   pack_check <D> <F> <T> <n> <missing> <weights.bin> <findex.bin> <tuples.bin>   ->  n*T uint32 leaf words (binary, stdout)
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

int main(int argc, char** argv) {
    if (argc < 9) return 2;
    Geom g;
    g.D = (uint32_t)atoi(argv[1]); const uint32_t F = (uint32_t)atoi(argv[2]), T = (uint32_t)atoi(argv[3]);
    const size_t n = (size_t)atoll(argv[4]);
    g.missing = (uint32_t)strtoul(argv[5], nullptr, 0);
    g.K = 1; g.S = 1; g.tuple_cls = F / 4;
    g.w_cls = (uint32_t)(((2ull << g.D) - 1 + 3) / 4); g.f_cls = (uint32_t)(((1ull << g.D) - 1 + 7) / 8);
    auto wl = slurp(argv[6]), fl = slurp(argv[7]), xs = slurp(argv[8]);
    PackedEnsemble pk;
    std::string msg;
    int rc = pack_ensemble(g, wl.data(), wl.size() / 16, fl.data(), fl.size() / 16, 0, 0, pk, msg);
    if (rc) { fprintf(stderr, "pack_ensemble: %d %s\n", rc, msg.c_str()); return 3; }
    const EnsembleShape& sh = pk.shape;
    if (sh.T != T) return 4;
    const uint32_t* X = reinterpret_cast<const uint32_t*>(xs.data());
    const int BV = sh.wide ? 4 : 2;
    std::vector<uint32_t> out(n * T);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t* x = X + i * F;
        for (uint32_t t = 0; t < T; ++t) {
            // top: byte offset o into the tree's 8-byte heap records, child = 2o + 8 + 8*right  (step_inc in dte_kernels.cuh)
            uint32_t o = 0;
            const uint2* tp = pk.top.data() + (size_t)t * sh.top_stride;
            for (uint32_t lvl = 0; lvl < sh.Dtop; ++lvl) {
                const uint2 nd = tp[o / 8];
                const uint32_t xv = x[nd.y & 0xFFFFu];
                uint32_t inc = ((int32_t)xv < (int32_t)nd.x) ? 8u : 16u;
                if (xv == g.missing) inc = nd.y >> 16;
                o = 2 * o + inc;
            }
            const uint32_t j = (o >> 3) - (sh.nb - 1);
            const uint4* rec = pk.bottom.data() + ((size_t)t * sh.nb + j) * BV;
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
            const bool r1 = (xp == g.missing) ? (mp != 0) : !((int32_t)xp < (int32_t)rec[0].x);
            const uint32_t thr = r1 ? rec[0].z : rec[0].y, xc = x[r1 ? fr : fl_], mc = r1 ? mr : ml;
            const bool r2 = (xc == g.missing) ? (mc != 0) : !((int32_t)xc < (int32_t)thr);
            out[i * T + t] = r1 ? (r2 ? leaves.w : leaves.z) : (r2 ? leaves.y : leaves.x);
        }
    }
    fwrite(out.data(), 4, out.size(), stdout);
    return 0;
}
