// opencv_fisheye x {none, digital_stretch} here; the three *view digital lenses are compiled in inst_opencv_fisheye_views.cu /
// inst_opencv_fisheye_hyper.cu so that the build parallelises (the pairs the reference pre-compiles:
// src/qt_gpu/compiled/compile_shaders.sh:6-27)
#include "kernel_registry.h"
namespace gf {
KernelFn gf_kernel_opencv_fisheye_superviews(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_opencv_fisheye_hyperview(int layout, int interp, KernelVariant v);
KernelFn gf_kernel_opencv_fisheye(int digital, int layout, int interp, KernelVariant v) {
    switch (digital) {
    case GF_LENS_NONE:             return pick_layout<GF_LENS_OPENCV_FISHEYE, GF_LENS_NONE>(layout, interp, v);
    case GF_LENS_GOPRO_SUPERVIEW:
    case GF_LENS_GOPRO6_SUPERVIEW: return gf_kernel_opencv_fisheye_superviews(digital, layout, interp, v);
    case GF_LENS_GOPRO_HYPERVIEW:  return gf_kernel_opencv_fisheye_hyperview(layout, interp, v);
    case GF_LENS_DIGITAL_STRETCH:  return pick_layout<GF_LENS_OPENCV_FISHEYE, GF_LENS_DIGITAL_STRETCH>(layout, interp, v);
    default: return nullptr;
    }
}
}
