// kernels_vol_ltree.cu -- the volume instantiations of k_shade with the light tree (EZRT_PARAM_VOLUMES with EZRT_PARAM_LIGHT_TREE):
// kernels_vol.cu's launcher with LTREE = true, launched by launch_shade through launch_shade_vol_ltree.
#define EZRT_KERNELS_LTREE
#define EZRT_VOL_LTREE true
#define EZRT_VOL_MEDIUM false
#define EZRT_VOL_LAUNCH launch_shade_vol_ltree
#include "kernels_vol.cu"
