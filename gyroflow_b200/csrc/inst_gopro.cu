// gopro x {none, gopro_warp} (src/qt_gpu/compiled/compile_shaders.sh:6-27)
#include "kernel_registry.h"
namespace gf {
KernelFn gf_kernel_gopro(int digital, int layout, int interp, KernelVariant v) {
    switch (digital) {
    case GF_LENS_NONE:       return pick_layout<GF_LENS_GOPRO, GF_LENS_NONE>(layout, interp, v);
    case GF_LENS_GOPRO_WARP: return pick_layout<GF_LENS_GOPRO, GF_LENS_GOPRO_WARP>(layout, interp, v);
    default: return nullptr;
    }
}
}
