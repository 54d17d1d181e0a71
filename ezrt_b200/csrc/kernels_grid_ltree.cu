// kernels_grid_ltree.cu -- the density-grid instantiations of k_shade with the light tree (EZRT_PARAM_MEDIUM_GRID with
// EZRT_PARAM_LIGHT_TREE): kernels_grid.cu's launcher with LTREE = true, launched by launch_shade through launch_shade_grid_ltree.
#define EZRT_KERNELS_LTREE
#define EZRT_GRID_LTREE true
#define EZRT_GRID_LAUNCH launch_shade_grid_ltree
#include "kernels_grid.cu"
