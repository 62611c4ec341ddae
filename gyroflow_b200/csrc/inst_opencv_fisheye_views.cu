// opencv_fisheye x {gopro_superview, gopro6_superview} (see inst_opencv_fisheye.cu)
#include "kernel_registry.h"
namespace gf {
KernelFn gf_kernel_opencv_fisheye_superviews(int digital, int layout, int interp, KernelVariant v) {
    if (digital == GF_LENS_GOPRO_SUPERVIEW) return pick_layout<GF_LENS_OPENCV_FISHEYE, GF_LENS_GOPRO_SUPERVIEW>(layout, interp, v);
    return pick_layout<GF_LENS_OPENCV_FISHEYE, GF_LENS_GOPRO6_SUPERVIEW>(layout, interp, v);
}
}
