// wgsl.h -- the WGSL front end of smr_register_wgsl_shader: a shader in the reference's dialect (its shader header,
// transformations/shader/validation/shader_header.wgsl, with a user vs_main and fs_main) translated to CUDA C++ for the
// NVRTC path of renderer.cpp.  Host C++ only.
#pragma once

#include <cstdint>
#include <optional>
#include <string>

#include "scene.h"

namespace smr {
namespace wgsl {

struct Translation {
    int status = 0;           // smr_status: SMR_OK, SMR_ERR_INVALID_ARGUMENT (CreateShaderError) or SMR_ERR_UNSUPPORTED
    std::string error;        // "line:col: what", for a status other than SMR_OK
    std::string cuda;         // the translated module, to be compiled after wgsl_rt.cuh
    std::optional<ShaderParamType> param_type;   // the type of the uniform at group(1) binding(0), if the module has one
    uint32_t uniform_size = 0;                   // its SizeOf in the uniform address space
};

// Lexes, parses, type-checks and validates `source` (validate_contains_header, UserBindingNotUniform), then emits CUDA
Translation translate(const std::string &source);

}  // namespace wgsl
}  // namespace smr
