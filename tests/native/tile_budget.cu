// Host-side report of the level kernel's tile geometry and shared-memory layout (stages.cuh, common.cuh): the sizes the
// shared-memory budget of two CTAs per SM is made of.  Built and run by tests/test_band_width.py (nvcc, host code only).
#include <cstddef>
#include <cstdio>

#include "stages.cuh"

int main() {
  using namespace dvo_b200;
  printf("tile_w %d\ntile_h %d\nwin_cols %d\nwin_rows %d\nstages %d\n", kTileW, kTileH, kWinCols, kWinRows, kStages);
  printf("rec_bytes %zu\nrec_stage_a_bytes %zu\n", (size_t)kRecF2 * sizeof(float2), (size_t)kRecP1 * sizeof(float2));
  printf("stage_buf %zu\ntile_pipe %zu\n", sizeof(StageBuf), sizeof(TilePipe));
  printf("seg_combine %zu\n", sizeof(SegCombineSmem));
  return 0;
}
