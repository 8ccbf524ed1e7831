// plan_check.cu — HOST-ONLY print of the launch planner's decisions (make_plan, kernel_name and phased_level in
// dte_device.cuh) on an H100's figures (132 SMs, 232,448 bytes of opt-in shared memory per block).  For every DTE_TUNE
// string below it sets the variable, parses it as an engine does, and prints one line per ensemble geometry and
// requested kernel variant:
//     <D> <F> <C> <variant> <phased level, -1 = off> <kernel name>
// tests/test_plan_table.py compares the output with tests/golden/plan_table.txt.xz.  Test infrastructure.
//   plan_check bin   the same grid for the binned walk (u8 tile, 4-byte tree tops): tests/golden/plan_table_binned.txt.xz
//   plan_check leaf  the same grid for the leaf walk (dt_walk_*_leaf): tests/golden/plan_table_leaf.txt.xz
#include "../distributed-decisiontrees_b200/csrc/dte_device.cuh"
#include <cstdio>
#include <cstdlib>
using namespace dte;

// the pins of the launch-plan tests and tools/gpu_sanitize.sh, dte_autotune's candidates, and pins the planner coerces
static const char* const kTunes[] = {
    "",
    "pair=1,ilp=8,stages=1", "pair=1,ilp=4,stages=2", "pair=2,stages=1", "pair=2,stages=2", "pair=4,stages=1",
    "pair=1,ilp=8,stages=2,warps=3", "pair=2,stages=1,warps=4", "pair=2,ilp=2,stages=2", "pair=2,stages=1,phased=1",
    "pair=1,ilp=8,stages=1,phased=1", "pair=4,stages=2,phased=1",
    "ilp=4,pair=2,stages=1,phased=1,warps=0", "ilp=4,pair=2,stages=1,phased=0,warps=0",
    "ilp=4,pair=2,stages=1,phased=1,warps=10", "ilp=4,pair=2,stages=1,phased=0,warps=10",
    "ilp=2,pair=4,stages=1,phased=1,warps=0", "ilp=2,pair=4,stages=1,phased=0,warps=0",
    "ilp=8,pair=1,stages=1,phased=0,warps=0", "ilp=8,pair=1,stages=2,phased=0,warps=0",
    "ilp=4,pair=1,stages=2,phased=0,warps=0", "ilp=2,pair=2,stages=2,phased=0,warps=0",
    "ilp=2,pair=2,stages=1,phased=0,warps=0",
    "ilp=8", "ilp=2", "ilp=4", "pair=2,ilp=8,stages=1", "pair=3,ilp=2", "ilp=16,pair=2", "stages=9", "warps=10",
    "phased=0", "phased=2",
};

int main(int argc, char** argv) {
    const char* kind = argc > 1 ? argv[1] : "";
    const Walk walk = !strcmp(kind, "bin") ? Walk::Binned : !strcmp(kind, "leaf") ? Walk::Leaf : Walk::Fp32;
    const uint32_t Fs[] = {4, 8, 32, 64, 96, 128, 192, 256, 384, 512, 516, 768, 1024, 1536, 1796, 1800, 2048};
    for (const char* s : kTunes) {
        setenv("DTE_TUNE", s, 1);
        Tune tune;
        parse_tune(tune);
        printf("DTE_TUNE=%s\n", s);
        for (uint32_t D = 1; D <= 15; ++D)
            for (uint32_t F : Fs)
                for (uint32_t C : {1u, 3u}) {
                    Dev d;
                    d.sm_count = 132;
                    d.smem_optin = 232448;
                    EnsembleShape& sh = d.shape;
                    sh.g.D = D;
                    sh.g.tuple_cls = F / 4;
                    sh.Dtop = std::max(D, 2u) - 2;
                    sh.top_stride = sh.nb = 1u << sh.Dtop;
                    sh.wide = F > 512;                   // a feature index >= 512 needs the wide bottom record
                    sh.C = C;
                    sh.gpc = 4;
                    sh.T = sh.cls_max = 32;
                    sh.Tpad = C * sh.gpc * 8;
                    for (int want = KERNEL_AUTO; want <= KERNEL_TILE_STAGED; ++want) {
                        char name[256];
                        kernel_name(d, tune, want, name, sizeof name, walk);
                        const auto pl = make_plan(d, tune, want, walk);
                        printf("%u %u %u %d %d %s\n", D, F, C, want, (int)phased_level(d, tune, pl), name);
                    }
                }
    }
    return 0;
}
