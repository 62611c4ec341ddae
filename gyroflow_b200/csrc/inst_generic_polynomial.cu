// generic_polynomial x {none, digital_stretch} (src/qt_gpu/compiled/compile_shaders.sh:6-27)
#include "kernel_registry.h"
namespace gf {
KernelFn gf_kernel_generic_polynomial(int digital, int layout, int interp, KernelVariant v) {
    switch (digital) {
    case GF_LENS_NONE:            return pick_layout<GF_LENS_GENERIC_POLYNOMIAL, GF_LENS_NONE>(layout, interp, v);
    case GF_LENS_DIGITAL_STRETCH: return pick_layout<GF_LENS_GENERIC_POLYNOMIAL, GF_LENS_DIGITAL_STRETCH>(layout, interp, v);
    default: return nullptr;
    }
}
}
