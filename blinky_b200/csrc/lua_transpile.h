// Lua -> C++/CUDA transpiler for lens scripts (SURVEY section 8f rank 1: "evaluate
// lens_inverse for all W*H pixels in parallel ... a Lua->CUDA/NVRTC transpile for
// closed-form lenses").
//
// Input: the compiled `lens_inverse` closure living in a minilua::State (with its
// upvalues and the globals it reads as they are RIGHT NOW).  Output: target-neutral
// C++ source for the function and everything it calls, against the small prelude
// returned by transpile_prelude().  The same source is compiled
//   * by NVRTC for sm_90a (product: the lensmap is evaluated on the GPU), and
//   * by g++ in the CPU test-suite, where it must reproduce the interpreter bit for
//     bit (same libm) — that is how the transpiler itself is pinned.
//
// Exactness on the GPU: +,-,*,/ and sqrt are IEEE in both worlds (NVRTC runs with
// --fmad=false); only libm functions (sin, atan2, pow, ...) may differ from glibc in
// the last bits.  The transpiler tracks statically which values are "tainted" by such
// calls and emits risk checks exactly where a tainted value meets a discontinuity:
// comparisons, floor/ceil/modf, array indexing, and (in the kernel) the final
// double->float conversion of the ray.  A pixel with any risk flag is re-evaluated by
// the exact host interpreter, so the finished lensmap is bit-identical by construction.
//
// Anything outside the supported subset (strings, nil-valued variables, closures
// created per call, recursion, ...) makes transpile_lens() fail with a reason and the
// caller falls back to the host evaluator.
#pragma once

#include <string>
#include <vector>

#include "minilua/minilua.h"

namespace blinky {

struct TranspileResult {
    bool ok = false;
    std::string error;       // why the script is not transpilable
    std::string source;      // definitions; entry point: bool lt_entry(Ctx &c, double a0, double a1, LtD *r)
    int num_functions = 0;
    int num_mutable = 0;     // script-level variables the lens assigns (become per-pixel state)
};

// names of the host-provided script functions (latlon_to_ray, ray_to_latlon, plate_to_ray)
// are resolved through the State's current globals; `numplates` plates are baked in for plate_to_ray.
//
// globe_plate (optional): the globe's globe_plate(x, y, z) is translated into the same unit — one
// function table (a helper both scripts call is emitted once), one set of constant tables and one set
// of script-level slots, since lens and globe share one Lua state.  The source then also defines
//   #define LT_HAS_GLOBE_PLATE 1
//   bool lt_globe_plate(Ctx &c, double x, double y, double z, int *plate)
// with the host's ray_to_plate_index semantics: false and *plate = -1 for no value / nil, otherwise the
// last value returned, converted like lua_tointeger (risk-flagged where that conversion is not certain).
// Without globe_plate the source is exactly what it was before.
TranspileResult transpile_lens(minilua::State &L, const minilua::Value &lens_inverse, const minilua::Value *globe_plate = nullptr);
// the same for lens_forward(x, y, z) -> x, y; entry point: bool lt_entry(Ctx &c, double a0, double a1, double a2, LtD *r)
TranspileResult transpile_lens_forward(minilua::State &L, const minilua::Value &lens_forward, const minilua::Value *globe_plate = nullptr);
// globe_plate alone: lt_init_mut, its functions and lt_globe_plate, without lt_entry
TranspileResult transpile_globe_plate(minilua::State &L, const minilua::Value &globe_plate);

// Support code the generated source needs.  cuda = true: __device__ functions; false: plain C++.
std::string transpile_prelude(bool cuda, bool noinline_user_functions = false);

}  // namespace blinky
