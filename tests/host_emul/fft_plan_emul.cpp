// Host build of the two-pass FFT's launch planner (fft_core.cuh: make_plane_plans, what csrc/fft.cu's rfft2 and irfft2
// launch with).  Usage: fft_plan_emul H W [H W ...]
// prints one line per plane and pass:  "H W rows|cols N lanes m np | radices"
//   N: template length (0 = runtime length), lanes: channels per CTA, m: Bluestein convolution length (0: none),
//   np: runtime passes (-1: none of the runtime plan, 0: a 1-point axis), radices: the runtime plan's passes.
#include <cstdio>
#include <cstdlib>

#include "../../lama_b200/csrc/fft_core.cuh"

using namespace ffcb::fftc;

static void print(int h, int w, const char* pass, const LaunchPlan& p) {
  printf("%d %d %s %d %d %d %d |", h, w, pass, p.N, p.lanes, p.bluestein ? p.m : 0, p.rp.np);
  for (int i = 0; i < p.rp.np; ++i) printf(" %d", p.rp.radix[i]);
  printf("\n");
}

int main(int argc, char** argv) {
  for (int i = 1; i + 1 < argc; i += 2) {
    const int h = atoi(argv[i]), w = atoi(argv[i + 1]);
    const PlanePlans pp = make_plane_plans(h, w);
    print(h, w, "rows", pp.rows);
    print(h, w, "cols", pp.cols);
  }
  return 0;
}
