// Host probe of the f-k filter's planner: which column and row route build_fk_hostplan picks for a shape, with the
// opt-in shared memory of an H100 (232 448 bytes per block).  Run it with no D4W_* variable in the environment to see
// the routes shapes reach by themselves.
// usage:
//   fk_route_probe plan NX NS [NX NS ...]   one line per shape: "NX NS" followed by route fields (see print_route), or
//                                           "NX NS error <message>"
//   fk_route_probe sweep NS LO HI           the same line for every NX in [LO, HI] the planner accepts
#include <cstdio>
#include <cstdlib>
#include <string>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
using namespace d4w;

static const size_t kSmem = 232448;

// Route fields, in order: scheme nc dual tma x1 x2 np ra rb pipe chunk_pairs t1 row_fused col_threads.
// scheme is d4w_fk_plan_info's code (0 single-level, 1 single-level TMA, 2 two-level, 3 pipelined two-level, 4 chirp-z);
// col_threads is the thread count d4w_fk_plan_create gives the single-level column kernels (D4W_COL_THREADS = 512,
// capped at D4W_COL_THREADS_R25 = 256 when a dual plan carries a radix above 16; 512 for chirp-z), which is also the
// template the launcher instantiates for schemes 0 and 1.
static void print_route(int nx, int ns) {
    FkHostPlan hp;
    std::string err;
    if (build_fk_hostplan(nx, ns, kSmem, hp, err)) { printf("%d %d error %s\n", nx, ns, err.c_str()); return; }
    const int scheme = hp.czt ? 4 : hp.pipe ? 3 : hp.two_level ? 2 : hp.tma ? 1 : 0;
    const int col_threads = hp.czt ? 512 : (hp.dual && hp.col_max_radix > 16) ? 256 : 512;
    printf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d\n", nx, ns, scheme, hp.nc, hp.dual, hp.tma, hp.x1, hp.x2,
           hp.two_level ? hp.np2 : 0, hp.fused_ra, hp.fused_rb, hp.pipe, hp.two_level ? hp.chunk_pairs : 0, hp.t1,
           hp.row_fused, col_threads);
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string cmd = argv[1];
    if (cmd == "plan") {
        for (int a = 2; a + 1 < argc; a += 2) print_route(std::atoi(argv[a]), std::atoi(argv[a + 1]));
        return 0;
    }
    if (cmd == "sweep" && argc == 5) {
        const int ns = std::atoi(argv[2]), lo = std::atoi(argv[3]), hi = std::atoi(argv[4]);
        for (int nx = lo; nx <= hi; ++nx) print_route(nx, ns);
        return 0;
    }
    return 2;
}
