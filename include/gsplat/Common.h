// Common.h -- drop-in replacement for the reference's gsplat/Common.h (the part callers see).
//
// The reference header (/root/reference/gsplat/Common.h:1-54) is included by
// include/core/camera.hpp:7 and by gsplat's own sources.  Callers outside gsplat/ only use
// `gsplat::CameraModelType`; the GLM typedefs and the CUB helper in the reference header are
// internals of its CUDA kernels.  This replacement keeps the public names and values and pulls
// GLM in only when it is actually installed, because the CUDA backend itself does not use GLM.
#pragma once

#include <algorithm>
#include <cstdint>

#if !defined(GSB_NO_GLM) && defined(__has_include)
#if __has_include(<glm/gtc/type_ptr.hpp>)
#include <glm/gtc/type_ptr.hpp>
#define GSB_HAVE_GLM 1
#endif
#endif

namespace gsplat {

// Argument checks with the reference's wording (Common.h:12-19): failures throw c10::Error.
#define CHECK_CUDA(x) TORCH_CHECK(x.is_cuda(), #x " must be a CUDA tensor")
#define CHECK_CONTIGUOUS(x) TORCH_CHECK(x.is_contiguous(), #x " must be contiguous")
#define CHECK_INPUT(x) \
    CHECK_CUDA(x);     \
    CHECK_CONTIGUOUS(x)
#define DEVICE_GUARD(_ten) const at::cuda::OptionalCUDAGuard device_guard(device_of(_ten));

#ifdef GSB_HAVE_GLM
    using vec2 = glm::vec<2, float>;
    using vec3 = glm::vec<3, float>;
    using vec4 = glm::vec<4, float>;
    using mat2 = glm::mat<2, 2, float>;
    using mat3 = glm::mat<3, 3, float>;
    using mat4 = glm::mat<4, 4, float>;
    using mat3x2 = glm::mat<3, 2, float>;
#endif

    // Camera model selector; values are part of the ABI (Common.h:46-50) and equal GSB_CAMERA_*.
    enum CameraModelType {
        PINHOLE = 0,
        ORTHO = 1,
        FISHEYE = 2,
    };

#define N_THREADS_PACKED 256
#define ALPHA_THRESHOLD (1.f / 255.f)

} // namespace gsplat
