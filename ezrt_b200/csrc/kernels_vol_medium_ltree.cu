// kernels_vol_medium_ltree.cu -- the volume instantiations with the medium and the light tree: kernels_vol.cu's launcher with
// MEDIUM = true and LTREE = true, launched by launch_shade through launch_shade_vol_medium_ltree.
#define EZRT_KERNELS_LTREE
#define EZRT_VOL_LTREE true
#define EZRT_VOL_MEDIUM true
#define EZRT_VOL_LAUNCH launch_shade_vol_medium_ltree
#include "kernels_vol.cu"
