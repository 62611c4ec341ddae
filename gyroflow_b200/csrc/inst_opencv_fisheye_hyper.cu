// opencv_fisheye x gopro_hyperview (see inst_opencv_fisheye.cu)
#include "kernel_registry.h"
namespace gf {
KernelFn gf_kernel_opencv_fisheye_hyperview(int layout, int interp, KernelVariant v) {
    return pick_layout<GF_LENS_OPENCV_FISHEYE, GF_LENS_GOPRO_HYPERVIEW>(layout, interp, v);
}
}
