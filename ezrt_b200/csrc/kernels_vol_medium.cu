// kernels_vol_medium.cu -- the volume instantiations with the medium (EZRT_PARAM_VOLUMES with EZRT_PARAM_MEDIUM, DESIGN.md section 21):
// kernels_vol.cu's launcher with MEDIUM = true (the homogeneous medium and the density grid), launched by launch_shade through
// launch_shade_vol_medium, and the k_nee<.., TRANS, MEDIUM, .., GRID> of launch_nee_vol_medium.
#define EZRT_VOL_LTREE false
#define EZRT_VOL_MEDIUM true
#define EZRT_VOL_LAUNCH launch_shade_vol_medium
#include "kernels_vol.cu"
