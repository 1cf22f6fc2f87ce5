// Host side of the H100 lens-warp path.  See fisheye_host.h.
//
// Numeric contract (what makes the lensmap bit-identical to the reference's):
// rays are float32 (`vec_t`, engine/include/mathlib.h:30) wherever the
// reference stores them in a vec3_t, everything a script computes is float64,
// float expressions are evaluated in float (x86-64, FLT_EVAL_METHOD 0) and this
// file is compiled with -ffp-contract=off and never with -ffast-math.
#include "fisheye_host.h"
#include "lua_transpile.h"
#include "parallel.h"

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <mutex>
#include <sstream>
#include <thread>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

using minilua::LuaError;
using minilua::State;
using minilua::Table;
using minilua::Value;
using minilua::ValueList;

namespace blinky {

// ---------------------------------------------------------------------------
// small float32 vector helpers with the engine's exact evaluation order
// (engine/common/mathlib.c:349-429, DotProduct macro mathlib.h:70)
// ---------------------------------------------------------------------------
namespace {

inline float dot3(const float a[3], const float b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

inline void madd3(const float a[3], float s, const float b[3], float out[3]) {
    out[0] = a[0] + s * b[0];
    out[1] = a[1] + s * b[1];
    out[2] = a[2] + s * b[2];
}

inline void cross3(const float a[3], const float b[3], float out[3]) {
    out[0] = a[1] * b[2] - a[2] * b[1];
    out[1] = a[2] * b[0] - a[0] * b[2];
    out[2] = a[0] * b[1] - a[1] * b[0];
}

inline void normalize3(float v[3]) {
    float len = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    len = static_cast<float>(std::sqrt(static_cast<double>(len)));
    if (len) {
        float inv = 1 / len;
        v[0] *= inv;
        v[1] *= inv;
        v[2] *= inv;
    }
}

// Quake's number grammar (engine/common/common.c Q_atof/Q_atoi): optional '-',
// 0x hex, 'c' character constants, decimals accumulated digit by digit and
// scaled by repeated division — no exponents.
double quake_atof(const char *s) {
    int sign = 1;
    if (*s == '-') {
        sign = -1;
        ++s;
    }
    double val = 0;
    if (s[0] == '0' && (s[1] == 'x' || s[1] == 'X')) {
        for (s += 2;; ++s) {
            int c = *s;
            if (c >= '0' && c <= '9') val = val * 16 + c - '0';
            else if (c >= 'a' && c <= 'f') val = val * 16 + c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') val = val * 16 + c - 'A' + 10;
            else return val * sign;
        }
    }
    if (s[0] == '\'') return sign * s[1];
    int decimal = -1, total = 0;
    for (;; ++s) {
        int c = *s;
        if (c == '.') {
            decimal = total;
            continue;
        }
        if (c < '0' || c > '9') break;
        val = val * 10 + c - '0';
        ++total;
    }
    if (decimal == -1) return val * sign;
    for (; total > decimal; --total) val /= 10;
    return val * sign;
}
inline float q_atof(const std::string &s) { return static_cast<float>(quake_atof(s.c_str())); }
inline int q_atoi(const std::string &s) {
    // Q_atoi: same grammar without the fraction
    const char *p = s.c_str();
    int sign = 1;
    if (*p == '-') {
        sign = -1;
        ++p;
    }
    int val = 0;
    if (p[0] == '0' && (p[1] == 'x' || p[1] == 'X')) {
        for (p += 2;; ++p) {
            int c = *p;
            if (c >= '0' && c <= '9') val = (val << 4) + c - '0';
            else if (c >= 'a' && c <= 'f') val = (val << 4) + c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') val = (val << 4) + c - 'A' + 10;
            else return val * sign;
        }
    }
    if (p[0] == '\'') return sign * p[1];
    for (;; ++p) {
        int c = *p;
        if (c < '0' || c > '9') return val * sign;
        val = val * 10 + c - '0';
    }
}

// console tokeniser: whitespace separated words, "quoted strings" kept whole
std::vector<std::string> tokenize(const std::string &line) {
    std::vector<std::string> out;
    size_t i = 0, n = line.size();
    while (i < n) {
        while (i < n && (line[i] == ' ' || line[i] == '\t' || line[i] == '\r')) ++i;
        if (i >= n || line[i] == '\n' || line[i] == ';') break;
        std::string tok;
        if (line[i] == '"') {
            ++i;
            while (i < n && line[i] != '"') tok.push_back(line[i++]);
            if (i < n) ++i;
        } else {
            while (i < n && !strchr(" \t\r\n;", line[i])) tok.push_back(line[i++]);
        }
        out.push_back(tok);
    }
    return out;
}

bool ieq(const std::string &a, const char *b) { return strcasecmp(a.c_str(), b) == 0; }

// lua_isnumber / lua_tonumber on a global
bool global_number(State &L, const char *name, double *out) { return L.get_global(name).to_number(out); }

}  // namespace

// One Lua state plus the function handles the reference keeps as registry refs.
struct FisheyeHost::Worker {
    State *L = nullptr;
    std::unique_ptr<State> owned;
    Value inverse, forward, globe_plate;
    bool has_globe_plate = false;
};

// ---------------------------------------------------------------------------
// construction: init_lua (fisheye.c:1222-1265) + F_Init's non-script defaults
// ---------------------------------------------------------------------------

static const char *kAliases =
    // fisheye.c:1230-1248 — the short names every lens script relies on
    "cos = math.cos\n"
    "sin = math.sin\n"
    "tan = math.tan\n"
    "asin = math.asin\n"
    "acos = math.acos\n"
    "atan = math.atan\n"
    "atan2 = math.atan2\n"
    "sinh = math.sinh\n"
    "cosh = math.cosh\n"
    "tanh = math.tanh\n"
    "log = math.log\n"
    "log10 = math.log10\n"
    "abs = math.abs\n"
    "sqrt = math.sqrt\n"
    "exp = math.exp\n"
    "pi = math.pi\n"
    "tau = math.pi*2\n"
    "pow = math.pow\n";

FisheyeHost::FisheyeHost() {
    memset(plates_, 0, sizeof plates_);
    memset(basepal_, 0, sizeof basepal_);
    lua_.reset(new State());
    // Lua's print() goes to stdout, as with the reference's stock Lua libraries
    // (tetra.lua:19 prints its fov); it is NOT a Con_Printf message.
    lua_->run(kAliases, "aliases");
    lua_->register_function("latlon_to_ray", &FisheyeHost::lua_latlon_to_ray, this);
    lua_->register_function("ray_to_latlon", &FisheyeHost::lua_ray_to_latlon, this);
    lua_->register_function("plate_to_ray", &FisheyeHost::lua_plate_to_ray, this);
    // F_Init :672 always runs "f_rubixgrid 10 4 1"
    rubix_numcells_ = 10;
    rubix_cell_ = 4;
    rubix_pad_ = 1;
}

FisheyeHost::~FisheyeHost() {
    fn_inverse_ = Value();
    fn_forward_ = Value();
    fn_globe_plate_ = Value();
}

void FisheyeHost::lua_print_sink(const char *text, void *ud) {
    // Lua's print() writes to stdout in the reference; route it to the message sink
    static_cast<FisheyeHost *>(ud)->print("%s", text);
}

void FisheyeHost::print(const char *fmt, ...) {
    char buf[2048];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    static std::mutex mu;  // worker threads of a parallel build may report errors
    std::lock_guard<std::mutex> g(mu);
    if (print_fn_) {
        print_fn_(buf, print_user_);
    } else {
        if (log_.size() < (1u << 20)) log_ += buf;
    }
}

// ---------------------------------------------------------------------------
// pure converters (fisheye.c:1184-1214) and their Lua wrappers (:1494-1537)
// ---------------------------------------------------------------------------

void FisheyeHost::latlon_to_ray(double lat, double lon, float ray[3]) {
    double clat = std::cos(lat);
    ray[0] = static_cast<float>(std::sin(lon) * clat);
    ray[1] = static_cast<float>(std::sin(lat));
    ray[2] = static_cast<float>(std::cos(lon) * clat);
}

void FisheyeHost::ray_to_latlon(const float ray[3], double *lat, double *lon) {
    *lon = std::atan2(static_cast<double>(ray[0]), static_cast<double>(ray[2]));
    float h2 = ray[0] * ray[0] + ray[2] * ray[2];  // float expression, :1195
    *lat = std::atan2(static_cast<double>(ray[1]), std::sqrt(static_cast<double>(h2)));
}

void FisheyeHost::plate_uv_to_ray(int plate, double u, double v, float ray[3]) const {
    const Plate &p = plates_[plate];
    u -= 0.5;
    v -= 0.5;
    v = -v;
    ray[0] = ray[1] = ray[2] = 0;
    madd3(ray, p.dist, p.forward, ray);
    madd3(ray, static_cast<float>(u), p.right, ray);  // VectorMA takes a float scale
    madd3(ray, static_cast<float>(v), p.up, ray);
    normalize3(ray);
}

static double arg_number(const Value *a, int n, int i, const char *fname) {
    double d;
    if (i > n || !a[i - 1].to_number(&d)) {
        std::ostringstream o;
        o << "bad argument #" << i << " to '" << fname << "' (number expected, got "
          << (i > n ? "no value" : State::type_name(a[i - 1])) << ")";
        throw LuaError(o.str());
    }
    return d;
}

void FisheyeHost::lua_latlon_to_ray(State &, const Value *a, int n, ValueList &out, void *) {
    double lat = arg_number(a, n, 1, "latlon_to_ray");
    double lon = arg_number(a, n, 2, "latlon_to_ray");
    float ray[3];
    latlon_to_ray(lat, lon, ray);  // through float32, like the vec3_t in :1498
    out.push_back(Value(static_cast<double>(ray[0])));
    out.push_back(Value(static_cast<double>(ray[1])));
    out.push_back(Value(static_cast<double>(ray[2])));
}

void FisheyeHost::lua_ray_to_latlon(State &, const Value *a, int n, ValueList &out, void *) {
    float ray[3] = {static_cast<float>(arg_number(a, n, 1, "ray_to_latlon")),
                    static_cast<float>(arg_number(a, n, 2, "ray_to_latlon")),
                    static_cast<float>(arg_number(a, n, 3, "ray_to_latlon"))};  // narrowed first, :1512
    double lat, lon;
    ray_to_latlon(ray, &lat, &lon);
    out.push_back(Value(lat));
    out.push_back(Value(lon));
}

void FisheyeHost::lua_plate_to_ray(State &, const Value *a, int n, ValueList &out, void *ud) {
    FisheyeHost *self = static_cast<FisheyeHost *>(ud);
    int plate = static_cast<int>(arg_number(a, n, 1, "plate_to_ray"));  // int plate_index = luaL_checknumber
    double u = arg_number(a, n, 2, "plate_to_ray");
    double v = arg_number(a, n, 3, "plate_to_ray");
    if (plate < 0 || plate >= self->numplates_) {
        out.push_back(Value());
        return;
    }
    float ray[3];
    self->plate_uv_to_ray(plate, u, v, ray);
    out.push_back(Value(static_cast<double>(ray[0])));
    out.push_back(Value(static_cast<double>(ray[1])));
    out.push_back(Value(static_cast<double>(ray[2])));
}

// ---------------------------------------------------------------------------
// palette (fisheye.c:835-908)
// ---------------------------------------------------------------------------

int FisheyeHost::find_closest_pal_index(int r, int g, int b) const {
    int best = 0, best_dist = 256 * 256 * 256;
    for (int i = 0; i < 256; ++i) {
        int dr = basepal_[3 * i] - r, dg = basepal_[3 * i + 1] - g, db = basepal_[3 * i + 2] - b;
        int dist = dr * dr + dg * dg + db * db;
        if (dist < best_dist) {  // first minimum wins
            best_dist = dist;
            best = i;
        }
    }
    return best;
}

void FisheyeHost::create_palmap() {
    // tint colours per plate: white, blue, red, yellow, magenta, cyan (:866-886)
    static const int kTint[kMaxPlates][3] = {{255, 255, 255}, {0, 0, 255}, {255, 0, 0},
                                             {255, 255, 0},   {255, 0, 255}, {0, 255, 255}};
    const int percent = 256 / 6;
    for (int j = 0; j < kMaxPlates; ++j)
        for (int i = 0; i < 256; ++i) {
            int c[3];
            for (int k = 0; k < 3; ++k) {
                int v = basepal_[3 * i + k];
                v += (percent * (kTint[j][k] - v)) >> 8;  // arithmetic shift of a possibly negative int
                c[k] = v < 0 ? 0 : (v > 255 ? 255 : v);
            }
            plates_[j].palette[i] = static_cast<uint8_t>(find_closest_pal_index(c[0], c[1], c[2]));
        }
}

void FisheyeHost::set_palette(const uint8_t palette[768]) {
    memcpy(basepal_, palette, 768);
    have_palette_ = true;
    create_palmap();
}

// ---------------------------------------------------------------------------
// console surface (fisheye.c:916-1176)
// ---------------------------------------------------------------------------

void FisheyeHost::set_zoom(int type, int fov) {
    // clear_zoom :1273-1278 then the type
    zoom_type_ = type;
    zoom_fov_ = (type == ZOOM_FOV || type == ZOOM_VFOV) ? fov : 0;
    zoom_changed_ = true;
}

void FisheyeHost::set_rubixgrid(int numcells, double cell, double pad) {
    rubix_numcells_ = numcells;
    rubix_cell_ = cell;
    rubix_pad_ = pad;
    lens_changed_ = true;  // :945
}

bool FisheyeHost::command(const std::string &line) {
    std::vector<std::string> argv = tokenize(line);
    if (argv.empty()) return true;
    const std::string &c = argv[0];
    const size_t argc = argv.size();

    if (ieq(c, "fisheye")) {  // cmd_fisheye :967-977
        if (argc < 2) {
            print("Currently: ");
            print("fisheye %d\n", fisheye_enabled_ ? 1 : 0);
            print("\nTry F_HELP for more options and commands.\n");
            return true;
        }
        fisheye_enabled_ = q_atoi(argv[1]) != 0;
        return true;
    }
    if (ieq(c, "f_help")) {  // cmd_help :1018-1030
        print("-----------------------------\n");
        print("Welcome to the FISHEYE ADDON!\n");
        print("-> fisheye 1    (ENABLE)\n");
        print("-> fisheye 0    (DISABLE)\n");
        print("\n");
        print("-> f_lens <tab>    (CHANGE LENS)\n");
        print("-> f_fov <degrees> (SET FOV)\n");
        print("\n");
        print("-> f_<tab>         (MORE COMMANDS)\n");
        print("-----------------------------\n");
        return true;
    }
    if (ieq(c, "f_rubix")) {  // cmd_rubix :933-937
        rubix_enabled_ = !rubix_enabled_;
        print("Rubix is %s\n", rubix_enabled_ ? "ON" : "OFF");
        return true;
    }
    if (ieq(c, "f_rubixgrid")) {  // cmd_rubixgrid :939-953
        if (argc == 4) {
            set_rubixgrid(static_cast<int>(q_atof(argv[1])), q_atof(argv[2]), q_atof(argv[3]));
        } else {
            print("RubixGrid <numcells> <cellsize> <padsize>\n");
            print("   numcells (default 10) = %d\n", rubix_numcells_);
            print("   cellsize (default  4) = %f\n", rubix_cell_);
            print("   padsize  (default  1) = %f\n", rubix_pad_);
        }
        return true;
    }
    if (ieq(c, "f_cover")) {
        set_zoom(ZOOM_COVER, 0);
        return true;
    }
    if (ieq(c, "f_contain")) {
        set_zoom(ZOOM_CONTAIN, 0);
        return true;
    }
    if (ieq(c, "f_fov") || ieq(c, "f_vfov")) {  // cmd_fov :1032-1044, cmd_vfov :1046-1058
        bool vertical = ieq(c, "f_vfov");
        if (argc < 2) {
            print(vertical ? "f_vfov <degrees>: set vertical FOV\n" : "f_fov <degrees>: set horizontal FOV\n");
            print("Zoom currently: ");  // print_zoom :1280-1291
            switch (zoom_type_) {
                case ZOOM_FOV: print("f_fov %d", zoom_fov_); break;
                case ZOOM_VFOV: print("f_vfov %d", zoom_fov_); break;
                case ZOOM_COVER: print("f_cover"); break;
                case ZOOM_CONTAIN: print("f_contain"); break;
                default: print("none");
            }
            print("\n");
            return true;
        }
        set_zoom(vertical ? ZOOM_VFOV : ZOOM_FOV, static_cast<int>(q_atof(argv[1])));
        return true;
    }
    if (ieq(c, "f_lens")) {  // cmd_lens :1061-1103
        if (argc < 2) {
            print("f_lens <name>: use a new lens\n");
            print("Currently: %s\n", lens_name_.c_str());
            return true;
        }
        cmd_lens(argv[1], nullptr);
        return true;
    }
    if (ieq(c, "f_globe")) {  // cmd_globe :1138-1161
        if (argc < 2) {
            print("f_globe <name>: use a new globe\n");
            print("Currently: %s\n", globe_name_.c_str());
            return true;
        }
        cmd_globe(argv[1], nullptr);
        return true;
    }
    if (ieq(c, "f_dumppal")) {  // cmd_dumppal :916-931
        FILE *f = fopen("palette", "w");
        if (!f) {
            print("could not open \"palette\" for writing\n");
            return true;
        }
        for (int i = 0; i < 256; ++i) fprintf(f, "%d, %d, %d,\n", basepal_[3 * i], basepal_[3 * i + 1], basepal_[3 * i + 2]);
        fclose(f);
        return true;
    }
    if (ieq(c, "f_shortcutkeys")) {  // cmd_shortcutkeys :979-1016 — key bindings belong to the engine
        shortcutkeys_enabled_ = !shortcutkeys_enabled_;
        static const char *kLens[] = {"panini", "stereographic", "hammer", "winkeltripel", "fisheye1",
                                      "mercator", "quincuncial", "cube", "debug"};
        static const char *kGlobeKeys[] = {"y", "u", "i", "o", "p"};
        static const char *kGlobes[] = {"cube", "cube_edge", "trism", "tetra", "fast"};
        char buf[128];
        if (shortcutkeys_enabled_) {
            print("Enabled Fisheye shortcut keys: 1-9 = Lenses, Y,U,I,O,P = Globes\n");
            if (exec_fn_) {
                for (int i = 0; i < 9; ++i) {
                    snprintf(buf, sizeof buf, "bind %d \"f_lens %s\"", i + 1, kLens[i]);
                    exec_fn_(buf, exec_user_);
                }
                for (int i = 0; i < 5; ++i) {
                    snprintf(buf, sizeof buf, "bind %s \"f_globe %s\"", kGlobeKeys[i], kGlobes[i]);
                    exec_fn_(buf, exec_user_);
                }
            }
        } else {
            print("Disabled Fisheye shortcut keys\n");
            if (exec_fn_) {
                for (int i = 1; i <= 8; ++i) {
                    snprintf(buf, sizeof buf, "bind %d \"impulse %d\"", i, i);
                    exec_fn_(buf, exec_user_);
                }
                exec_fn_("unbind 9", exec_user_);
                for (int i = 0; i < 5; ++i) {
                    snprintf(buf, sizeof buf, "unbind %s", kGlobeKeys[i]);
                    exec_fn_(buf, exec_user_);
                }
            }
        }
        return true;
    }
    if (ieq(c, "f_saveglobe")) {  // cmd_saveglobe :1120-1136
        if (argc < 2) {
            print("f_saveglobe <name> [full flag=0]: screenshot the globe plates\n");
            return true;
        }
        save_name_ = argv[1].substr(0, 31);
        save_with_margins_ = argc >= 3 ? q_atoi(argv[2]) : 0;
        save_pending_ = true;
        return true;
    }
    return false;
}

bool FisheyeHost::cmd_lens(const std::string &name, const std::string *source) {
    lens_changed_ = true;
    lens_name_ = name.substr(0, 49);  // char name[50]
    lens_from_source_ = source != nullptr;
    if (source) lens_source_ = *source;
    print("f_lens %s", lens_name_.c_str());
    lens_valid_ = load_lens();
    if (!lens_valid_) {
        lens_name_.clear();
        print("not a valid lens\n");
    }
    // run the script's `onload` command if it is a string (:1087-1102)
    Value onload = lua_->get_global("onload");
    if (onload.is_string() || onload.is_number()) {  // lua_isstring accepts numbers
        onload_ = State::tostring(onload);
        if (exec_fn_) exec_fn_(onload_.c_str(), exec_user_);
        else command(onload_);
        print("; %s\n", onload_.c_str());
    } else {
        onload_.clear();
        print("\n");
    }
    return lens_valid_;
}

bool FisheyeHost::cmd_globe(const std::string &name, const std::string *source) {
    globe_changed_ = true;
    globe_name_ = name.substr(0, 49);
    globe_from_source_ = source != nullptr;
    if (source) globe_source_ = *source;
    print("f_globe %s\n", globe_name_.c_str());
    globe_valid_ = load_globe();
    if (!globe_valid_) {
        globe_name_.clear();
        print("not a valid globe\n");
    }
    return globe_valid_;
}

std::string FisheyeHost::write_config() const {
    char buf[512];
    std::string out;
    snprintf(buf, sizeof buf, "fisheye %d\n", fisheye_enabled_ ? 1 : 0);
    out += buf;
    snprintf(buf, sizeof buf, "f_lens \"%s\"\n", lens_name_.c_str());
    out += buf;
    snprintf(buf, sizeof buf, "f_globe \"%s\"\n", globe_name_.c_str());
    out += buf;
    snprintf(buf, sizeof buf, "f_rubixgrid %d %f %f\n", rubix_numcells_, rubix_cell_, rubix_pad_);
    out += buf;
    switch (zoom_type_) {
        case ZOOM_FOV: snprintf(buf, sizeof buf, "f_fov %d\n", zoom_fov_); out += buf; break;
        case ZOOM_VFOV: snprintf(buf, sizeof buf, "f_vfov %d\n", zoom_fov_); out += buf; break;
        case ZOOM_COVER: out += "f_cover\n"; break;
        case ZOOM_CONTAIN: out += "f_contain\n"; break;
        default: break;
    }
    return out;
}

// ---------------------------------------------------------------------------
// globe export (fisheye.c:1396-1486)
// ---------------------------------------------------------------------------

std::vector<uint8_t> FisheyeHost::plate_pcx(const uint8_t *faces, int plate, bool with_margins) {
    const int ps = platesize_;
    std::vector<uint8_t> out(128, 0);  // pcx_t header (engine/NQ/client.h:377-391), zero-filled
    auto put16 = [&](size_t at, int v) {
        out[at] = static_cast<uint8_t>(v & 0xff);
        out[at + 1] = static_cast<uint8_t>((v >> 8) & 0xff);
    };
    out[0] = 0x0a;  // manufacturer
    out[1] = 5;     // version: 256 colours
    out[2] = 1;     // encoding
    out[3] = 8;     // bits per pixel
    put16(8, ps - 1);   // xmax
    put16(10, ps - 1);  // ymax
    put16(12, ps);      // hres
    put16(14, ps);      // vres
    out[65] = 1;        // colour planes
    put16(66, ps);      // bytes per line
    put16(68, 2);       // palette type
    Worker w;
    w.L = lua_.get();
    w.globe_plate = fn_globe_plate_;
    w.has_globe_plate = fn_globe_plate_.is_function();
    const uint8_t *data = faces + static_cast<size_t>(plate) * ps * ps;
    out.reserve(128 + static_cast<size_t>(ps) * ps * 2 + 769);
    for (int i = 0; i < ps; ++i) {
        double v = static_cast<double>(i) / ps;
        for (int j = 0; j < ps; ++j) {
            double u = static_cast<double>(j) / ps;
            uint8_t col = *data++;
            if (!with_margins) {
                float ray[3];
                plate_uv_to_ray(plate, u, v, ray);
                int owner;
                try {
                    owner = ray_to_plate_index(w, ray);
                } catch (LuaError &) {
                    owner = -1;
                }
                if (owner != plate) col = 0xFE;
            }
            if ((col & 0xc0) == 0xc0) out.push_back(0xc1);  // escape, as the reference's "uncompressed" RLE does
            out.push_back(col);
        }
    }
    out.push_back(0x0c);
    out.insert(out.end(), basepal_, basepal_ + 768);
    return out;
}

bool FisheyeHost::save_globe(const uint8_t *faces, const std::string &dir) {
    save_pending_ = false;
    bool ok = true;
    for (int i = 0; i < numplates_; ++i) {
        char name[64];
        snprintf(name, sizeof name, "%s%d.pcx", save_name_.c_str(), i);
        std::vector<uint8_t> pcx = plate_pcx(faces, i, save_with_margins_ != 0);
        std::string path = dir.empty() ? std::string(name) : dir + "/" + name;
        FILE *f = fopen(path.c_str(), "wb");
        if (f) {
            fwrite(pcx.data(), 1, pcx.size(), f);
            fclose(f);
        } else {
            ok = false;
        }
        print("Wrote %s\n", name);
    }
    return ok;
}

// ---------------------------------------------------------------------------
// script loading (fisheye.c:1659-1913)
// ---------------------------------------------------------------------------

void FisheyeHost::clear_lens_vars() {
    static const char *kVars[] = {"map", "max_fov", "max_vfov", "lens_width", "lens_height",
                                  "lens_inverse", "lens_forward", "onload"};
    for (const char *v : kVars) lua_->set_global(v, Value());
    lua_->set_global("numplates", Value(static_cast<double>(numplates_)));
}

void FisheyeHost::clear_globe_vars() {
    lua_->set_global("plates", Value());
    lua_->set_global("globe_plate", Value());
    numplates_ = 0;
}

bool FisheyeHost::run_script(const std::string &kind, const std::string &name, const std::string *source) {
    Value chunk;
    try {
        if (source) {
            chunk = lua_->load(*source, name + ".lua");
        } else {
            std::string path = basedir_ + "/lua-scripts/" + kind + "/" + name + ".lua";
            std::ifstream probe(path, std::ios::binary);
            if (!probe) {
                print("could not loadfile (%d) \nERROR: cannot open %s", 7, path.c_str());
                return false;
            }
            chunk = lua_->load_file(path);
        }
    } catch (LuaError &e) {
        print("could not loadfile (%d) \nERROR: %s", 3, e.what());
        return false;
    }
    try {
        ValueList out;
        lua_->call(chunk, nullptr, 0, out);
    } catch (LuaError &e) {
        print("could not pcall (%d) \nERROR: %s", 2, e.what());
        return false;
    }
    return true;
}

bool FisheyeHost::load_lens() {
    clear_lens_vars();
    if (!run_script("lenses", lens_name_, lens_from_source_ ? &lens_source_ : nullptr)) return false;

    map_type_ = MAP_NONE;
    fn_inverse_ = Value();
    fn_forward_ = Value();
    Value inv = lua_->get_global("lens_inverse");
    if (inv.is_function()) {
        fn_inverse_ = inv;
        map_type_ = MAP_INVERSE;
    }
    Value fwd = lua_->get_global("lens_forward");
    if (fwd.is_function()) {
        fn_forward_ = fwd;
        if (map_type_ == MAP_NONE) map_type_ = MAP_FORWARD;
    }
    Value map = lua_->get_global("map");
    if (map.is_string() || map.is_number()) {
        std::string m = State::tostring(map);
        if (m == "lens_inverse") map_type_ = MAP_INVERSE;
        else if (m == "lens_forward") map_type_ = MAP_FORWARD;
        else {
            print("Unsupported map function: %s\n", m.c_str());
            return false;
        }
    }
    double d;
    max_fov_ = global_number(*lua_, "max_fov", &d) ? static_cast<int>(d) : 0;
    max_vfov_ = global_number(*lua_, "max_vfov", &d) ? static_cast<int>(d) : 0;
    lens_width_ = global_number(*lua_, "lens_width", &d) ? d : 0;
    lens_height_ = global_number(*lua_, "lens_height", &d) ? d : 0;
    return true;
}

bool FisheyeHost::load_globe() {
    clear_globe_vars();
    if (!run_script("globes", globe_name_, globe_from_source_ ? &globe_source_ : nullptr)) return false;

    fn_globe_plate_ = Value();
    Value gp = lua_->get_global("globe_plate");
    if (gp.is_function()) fn_globe_plate_ = gp;

    Value pv = lua_->get_global("plates");
    if (!pv.is_table() || static_cast<Table *>(pv.obj())->length() < 1) {
        print("plates must be an array of one or more elements\n");
        return false;
    }
    Table *plates = static_cast<Table *>(pv.obj());
    int i = 0;
    size_t pos = 0;
    Value key, val;
    // lua_next order: array part first, in index order (:1796)
    while (plates->next(&pos, &key, &val)) {
        if (i >= kMaxPlates) {
            // the reference has no bound check here and overruns plates[]; refuse instead
            print("plates: more than %d plates are not supported\n", kMaxPlates);
            return false;
        }
        Plate &p = plates_[i];
        Table *pt = val.is_table() ? static_cast<Table *>(val.obj()) : nullptr;
        for (int which = 0; which < 2; ++which) {  // 1 = forward, 2 = up
            Value vec = pt ? pt->get_int(which + 1) : Value();
            if (!vec.is_table() || static_cast<Table *>(vec.obj())->length() != 3) {
                print("plate %d: %s vector is not a 3d vector\n", i + 1, which == 0 ? "forward" : "up");
                return false;
            }
            Table *vt = static_cast<Table *>(vec.obj());
            for (int j = 0; j < 3; ++j) {
                double d;
                if (!vt->get_int(j + 1).to_number(&d)) {
                    print("plate %d: %s vector: element %d not a number\n", i + 1, which == 0 ? "forward" : "up", j + 1);
                    return false;
                }
                (which == 0 ? p.forward : p.up)[j] = static_cast<float>(d);
            }
        }
        cross3(p.up, p.forward, p.right);  // :1849
        cross3(p.forward, p.right, p.up);  // :1850 — not normalised, as in the reference
        double fov_deg = 0;
        Value fv = pt->get_int(3);
        if (!fv.to_number(&fov_deg)) {
            print("plate %d: fov not a number\n", i + 1);
            fov_deg = 0;
        }
        p.fov = static_cast<float>(fov_deg * M_PI / 180);
        if (p.fov <= 0) {
            print("plate %d: fov must > 0\n", i + 1);
            return false;
        }
        p.dist = static_cast<float>(0.5 / std::tan(static_cast<double>(p.fov / 2)));
        ++i;
    }
    numplates_ = i;
    return true;
}

// ---------------------------------------------------------------------------
// Lua -> C calls (fisheye.c:1545-1651)
// ---------------------------------------------------------------------------

int FisheyeHost::call_inverse(Worker &w, double x, double y, float ray[3]) {
    Value args[2] = {Value(x), Value(y)};
    ValueList ret;
    w.L->call(w.inverse, args, 2, ret);  // LuaError propagates to the builder
    if (ret.size() == 3) {
        double a, b, c;
        if (ret[0].to_number(&a) && ret[1].to_number(&b) && ret[2].to_number(&c)) {
            ray[0] = static_cast<float>(a);
            ray[1] = static_cast<float>(b);
            ray[2] = static_cast<float>(c);
            normalize3(ray);
            return 1;
        }
        print("lens_inverse returned a non-number value for x,y,z\n");
        return -1;
    }
    if (ret.size() == 1) {
        if (ret[0].is_nil()) return 0;
        print("lens_inverse returned a single non-nil value\n");
        return -1;
    }
    print("lens_inverse returned %d values instead of 3\n", ret.size());
    return -1;
}

int FisheyeHost::call_forward(Worker &w, const float ray[3], double *x, double *y) {
    Value args[3] = {Value(static_cast<double>(ray[0])), Value(static_cast<double>(ray[1])), Value(static_cast<double>(ray[2]))};
    ValueList ret;
    w.L->call(w.forward, args, 3, ret);
    if (ret.size() == 2) {
        if (ret[0].to_number(x) && ret[1].to_number(y)) return 1;
        print("lens_forward returned a non-number value for x,y\n");
        return -1;
    }
    if (ret.size() == 1) {
        if (ret[0].is_nil()) return 0;
        print("lens_forward returned a single non-nil value\n");
        return -1;
    }
    print("lens_forward returned %d values instead of 2\n", ret.size());
    return -1;
}

bool FisheyeHost::lens_device_source(bool cuda, std::string *source, std::string *why, bool forward) {
    const Value &fn = forward ? fn_forward_ : fn_inverse_;
    if (!fn.is_function()) {
        *why = forward ? "the lens has no lens_forward" : "the lens has no lens_inverse";
        return false;
    }
    if (fn_globe_plate_.is_function()) {
        *why = "the globe selects plates with a script function (globe_plate)";
        return false;
    }
    TranspileResult r = forward ? transpile_lens_forward(*lua_, fn) : transpile_lens(*lua_, fn);
    if (!r.ok) {
        *why = r.error;
        return false;
    }
    // BLINKY_LENS_NOINLINE=1: script functions become real device calls (faster NVRTC, slower kernel)
    const char *ni = getenv("BLINKY_LENS_NOINLINE");
    *source = transpile_prelude(cuda, ni && ni[0] == '1') + r.source;
    return true;
}

int FisheyeHost::lens_inverse(double x, double y, double out[3]) {
    if (!fn_inverse_.is_function()) return -2;
    Value args[2] = {Value(x), Value(y)};
    ValueList ret;
    try {
        lua_->call(fn_inverse_, args, 2, ret);
    } catch (LuaError &e) {
        print("%s\n", e.what());
        return -3;
    }
    if (ret.size() == 3 && ret[0].to_number(&out[0]) && ret[1].to_number(&out[1]) && ret[2].to_number(&out[2])) return 1;
    if (ret.size() == 1 && ret[0].is_nil()) return 0;
    return -1;
}

int FisheyeHost::lens_forward(double rx, double ry, double rz, double *x, double *y) {
    if (!fn_forward_.is_function()) return -2;
    Value args[3] = {Value(rx), Value(ry), Value(rz)};
    ValueList ret;
    try {
        lua_->call(fn_forward_, args, 3, ret);
    } catch (LuaError &e) {
        print("%s\n", e.what());
        return -3;
    }
    if (ret.size() == 2 && ret[0].to_number(x) && ret[1].to_number(y)) return 1;
    if (ret.size() == 1 && ret[0].is_nil()) return 0;
    return -1;
}

// ---------------------------------------------------------------------------
// zoom (fisheye.c:1293-1386)
// ---------------------------------------------------------------------------

bool FisheyeHost::calc_zoom() {
    scale_ = -1;
    if (zoom_type_ == ZOOM_FOV || zoom_type_ == ZOOM_VFOV) {
        if (max_fov_ <= 0 || max_vfov_ <= 0) {
            print("max_fov & max_vfov not specified, try \"f_cover\"\n");
            return false;
        } else if (zoom_type_ == ZOOM_FOV && zoom_fov_ > max_fov_) {
            print("fov must be less than %d\n", max_fov_);
            return false;
        } else if (zoom_type_ == ZOOM_VFOV && zoom_fov_ > max_vfov_) {
            print("vfov must be less than %d\n", max_vfov_);
            return false;
        }
        if (!fn_forward_.is_function()) {
            print("Please specify a forward mapping function in your script for FOV scaling\n");
            return false;
        }
        Worker w;
        w.L = lua_.get();
        w.forward = fn_forward_;
        float ray[3];
        double x = 0, y = 0;
        double fovr = zoom_fov_ * M_PI / 180;
        int status;
        if (zoom_type_ == ZOOM_FOV) latlon_to_ray(0, fovr * 0.5, ray);
        else latlon_to_ray(fovr * 0.5, 0, ray);
        try {
            status = call_forward(w, ray, &x, &y);
        } catch (LuaError &e) {
            print("%s\n", e.what());
            status = -1;
        }
        // the reference tests the status for truth (:1322), so -1 would use
        // garbage; only a real (x,y) is accepted here
        if (status != 1) {
            print("ray_to_xy did not return a valid r value for determining FOV scale\n");
            return false;
        }
        scale_ = zoom_type_ == ZOOM_FOV ? x / (width_px_ * 0.5) : y / (height_px_ * 0.5);
    } else if (zoom_type_ == ZOOM_CONTAIN || zoom_type_ == ZOOM_COVER) {
        double fit_w = lens_width_ / width_px_;
        double fit_h = lens_height_ / height_px_;
        bool have_w = lens_width_ > 0, have_h = lens_height_ > 0;
        if (!have_w && have_h) {
            scale_ = fit_h;
        } else if (have_w && !have_h) {
            scale_ = fit_w;
        } else if (!have_w && !have_h) {
            print("neither lens_height nor lens_width are valid/specified.  Try f_fov instead.\n");
            return false;
        } else {
            double lens_aspect = lens_width_ / lens_height_;
            double screen_aspect = static_cast<double>(width_px_) / height_px_;
            bool lens_wider = lens_aspect > screen_aspect;
            if (zoom_type_ == ZOOM_CONTAIN) scale_ = lens_wider ? fit_w : fit_h;
            else scale_ = lens_wider ? fit_h : fit_w;
        }
    }
    if (scale_ <= 0) {
        print("init returned a scale of %f, which is  <= 0\n", scale_);
        return false;
    }
    return true;
}

// ---------------------------------------------------------------------------
// globe getters and lensmap setters (fisheye.c:1922-2066)
// ---------------------------------------------------------------------------

int FisheyeHost::ray_to_plate_index(Worker &w, const float ray[3]) {
    if (w.has_globe_plate) {  // user-defined plate selection (:2027-2033, :1634-1651)
        Value args[3] = {Value(static_cast<double>(ray[0])), Value(static_cast<double>(ray[1])), Value(static_cast<double>(ray[2]))};
        ValueList ret;
        w.L->call(w.globe_plate, args, 3, ret);
        double d;
        if (ret.size() == 0 || !ret[ret.size() - 1].to_number(&d)) return -1;  // lua_isnumber(-1)
        return static_cast<int>(static_cast<ptrdiff_t>(d));                    // lua_tointeger
    }
    int best = 0;
    double best_dp = -2;
    for (int i = 0; i < numplates_; ++i) {
        double dp = dot3(ray, plates_[i].forward);  // float dot product, widened
        if (dp > best_dp) {                          // strict: lowest index wins ties; NaN never wins
            best_dp = dp;
            best = i;
        }
    }
    return best;
}

bool FisheyeHost::ray_to_plate_uv(int plate, const float ray[3], double *u, double *v) const {
    const Plate &p = plates_[plate];
    double x = dot3(p.right, ray);
    double y = dot3(p.up, ray);
    double z = dot3(p.forward, ray);
    double dist = 0.5 / std::tan(static_cast<double>(p.fov / 2));  // float halving, double tan (:2060)
    *u = x / z * dist + 0.5;
    *v = -y / z * dist + 0.5;
    return *u >= 0 && *u <= 1 && *v >= 0 && *v <= 1;
}

void FisheyeHost::set_from_plate(int lx, int ly, int px, int py, int plate, int *display) {
    if (lx < 0 || lx >= width_px_ || ly < 0 || ly >= height_px_) return;
    if (px < 0 || px >= platesize_ || py < 0 || py >= platesize_) return;
    display[plate] = 1;
    size_t at = static_cast<size_t>(lx) + static_cast<size_t>(ly) * width_px_;
    idx_[at] = plate * platesize_ * platesize_ + px + py * platesize_;
    // rubix grid (:1922-1960): cells get the plate's tint, the padding between
    // them keeps whatever tint the pixel already had
    double block = rubix_pad_ + rubix_cell_;
    double units = rubix_numcells_ * block + rubix_pad_;
    double unit_px = static_cast<double>(platesize_) / units;
    double ux = static_cast<double>(px) / unit_px;
    double uy = static_cast<double>(py) / unit_px;
    bool ongrid = std::fmod(ux, block) < rubix_pad_ || std::fmod(uy, block) < rubix_pad_;
    if (!ongrid) tint_[at] = static_cast<uint8_t>(plate);
}

void FisheyeHost::set_from_ray(Worker &w, int lx, int ly, const float ray[3], int *display) {
    int plate = ray_to_plate_index(w, ray);
    if (plate < 0) return;
    if (plate >= kMaxPlates) return;  // reference would index plates[] out of range
    double u, v;
    if (!ray_to_plate_uv(plate, ray, &u, &v)) return;
    int px = static_cast<int>(u * platesize_);
    int py = static_cast<int>(v * platesize_);
    set_from_plate(lx, ly, px, py, plate, display);
}

// ---------------------------------------------------------------------------
// inverse builder (fisheye.c:2084-2124)
// ---------------------------------------------------------------------------

int FisheyeHost::build_inverse_rows(Worker &w, int y_begin, int y_end, int *display) {
    for (int ly = y_end - 1; ly >= y_begin; --ly) {
        double y = -(ly - height_px_ / 2) * scale_;
        for (int lx = 0; lx < width_px_; ++lx) {
            double x = (lx - width_px_ / 2) * scale_;
            float ray[3];
            int status = call_inverse(w, x, y, ray);
            if (status == 0) continue;
            if (status == -1) return -1;
            set_from_ray(w, lx, ly, ray, display);
        }
    }
    return 0;
}

int FisheyeHost::build_inverse_pixels(Worker &w, const int32_t *pixels, size_t n, int *display) {
    for (size_t i = 0; i < n; ++i) {
        const int ly = pixels[i] / width_px_, lx = pixels[i] % width_px_;
        double y = -(ly - height_px_ / 2) * scale_;
        double x = (lx - width_px_ / 2) * scale_;
        float ray[3];
        int status = call_inverse(w, x, y, ray);
        if (status == 0) continue;
        if (status == -1) return -1;
        set_from_ray(w, lx, ly, ray, display);
    }
    return 0;
}

template <class F>
int FisheyeHost::run_inverse_workers(int threads, int nitems, int *display, F item) {
    int rc = 0;
    if (threads <= 1 || nitems <= 1) {
        Worker w;
        w.L = lua_.get();
        w.inverse = fn_inverse_;
        w.globe_plate = fn_globe_plate_;
        w.has_globe_plate = fn_globe_plate_.is_function();
        try {
            for (int i = 0; i < nitems && rc == 0; ++i) rc = item(w, i, display);
        } catch (LuaError &e) {
            print("%s\n", e.what());
            rc = -1;
        }
        return rc;
    }
    // Cloned Lua states.  The handles are parked in globals so that State::clone()
    // carries them over to each worker.
    lua_->set_global("__blinky_inverse", fn_inverse_);
    lua_->set_global("__blinky_globe_plate", fn_globe_plate_);
    std::vector<Worker> workers(static_cast<size_t>(threads));
    for (auto &w : workers) {
        w.owned = lua_->clone();
        w.L = w.owned.get();
        w.inverse = w.L->get_global("__blinky_inverse");
        w.globe_plate = w.L->get_global("__blinky_globe_plate");
        w.has_globe_plate = w.globe_plate.is_function();
    }
    lua_->set_global("__blinky_inverse", Value());
    lua_->set_global("__blinky_globe_plate", Value());
    std::atomic<int> next_item(0);
    std::atomic<int> failed(0);
    std::vector<std::array<int, kMaxPlates>> disp(static_cast<size_t>(threads));
    for (auto &d : disp) d.fill(0);
    std::vector<std::string> errors(static_cast<size_t>(threads));
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) {
        pool.emplace_back([&, t]() {
            Worker &w = workers[static_cast<size_t>(t)];
            for (;;) {
                int i = next_item.fetch_add(1);
                if (i >= nitems || failed.load()) break;
                try {
                    if (item(w, i, disp[static_cast<size_t>(t)].data()) != 0) failed.store(1);
                } catch (LuaError &e) {
                    errors[static_cast<size_t>(t)] = e.what();
                    failed.store(1);
                }
            }
        });
    }
    for (auto &th : pool) th.join();
    // release worker handles before their states die
    for (auto &w : workers) {
        w.inverse = Value();
        w.globe_plate = Value();
    }
    for (auto &d : disp)
        for (int i = 0; i < kMaxPlates; ++i) display[i] |= d[static_cast<size_t>(i)];
    if (failed.load()) {
        for (auto &e : errors)
            if (!e.empty()) print("%s\n", e.c_str());
        rc = -1;
    }
    return rc;
}

LensBuildParams FisheyeHost::device_params() const {
    LensBuildParams p;
    memset(&p, 0, sizeof p);
    p.width = width_px_;
    p.height = height_px_;
    p.platesize = platesize_;
    p.numplates = numplates_;
    p.scale = scale_;
    // rubix grid geometry exactly as set_from_plate derives it
    p.rubix_block = rubix_pad_ + rubix_cell_;
    p.rubix_pad = rubix_pad_;
    const double units = rubix_numcells_ * p.rubix_block + rubix_pad_;
    p.rubix_unit_px = static_cast<double>(platesize_) / units;
    for (int i = 0; i < numplates_; ++i) {
        const Plate &pl = plates_[i];
        p.uv_dist[i] = 0.5 / std::tan(static_cast<double>(pl.fov / 2));
        for (int k = 0; k < 3; ++k) {
            p.plates[i].forward[k] = pl.forward[k];
            p.plates[i].right[k] = pl.right[k];
            p.plates[i].up[k] = pl.up[k];
        }
        p.plates[i].dist = pl.dist;
    }
    return p;
}

int FisheyeHost::build_inverse_device(int *display, std::string *why) {
    std::string src;
    if (!lens_device_source(true, &src, why)) return 1;
    const LensBuildParams p = device_params();
    const size_t area = idx_.size();
    std::vector<uint32_t> cand(area);
    if (!device_builder_->build(src, p, cand.data(), why)) return 1;

    std::vector<int32_t> undecided;
    {
        const int ps2 = platesize_ * platesize_;
        const int rows_per = 16;
        const int nchunks = (height_px_ + rows_per - 1) / rows_per;
        std::vector<std::vector<int32_t>> und(static_cast<size_t>(nchunks));
        std::vector<std::array<int, kMaxPlates>> disp(static_cast<size_t>(nchunks));
        parallel_for(nchunks, fallback_threads_, [&](int ch) {
            std::array<int, kMaxPlates> &dp = disp[static_cast<size_t>(ch)];
            dp.fill(0);
            const size_t b = static_cast<size_t>(ch) * rows_per * width_px_;
            const size_t e = std::min(area, b + static_cast<size_t>(rows_per) * width_px_);
            for (size_t at = b; at < e; ++at) {
                const uint32_t c = cand[at];
                if (c & kCandRisk) {
                    und[static_cast<size_t>(ch)].push_back(static_cast<int32_t>(at));
                } else if (c & kCandValid) {
                    const int32_t ix = static_cast<int32_t>(c & 0x0FFFFFFFu);
                    int plate = 0;
                    for (int32_t lim = ps2; ix >= lim; lim += ps2) ++plate;  // <= 5 steps, cheaper than a division
                    idx_[at] = ix;
                    dp[static_cast<size_t>(plate)] = 1;
                    if (!(c & kCandOnGrid)) tint_[at] = static_cast<uint8_t>(plate);
                }
            }
        });
        for (int ch = 0; ch < nchunks; ++ch) {
            undecided.insert(undecided.end(), und[static_cast<size_t>(ch)].begin(), und[static_cast<size_t>(ch)].end());
            for (int i = 0; i < kMaxPlates; ++i) display[i] |= disp[static_cast<size_t>(ch)][static_cast<size_t>(i)];
        }
    }
    // the interpreter decides what the device could not
    const int chunk = 256;
    const int nitems = static_cast<int>((undecided.size() + chunk - 1) / chunk);
    const int threads = undecided.size() >= 4096 ? fallback_threads_ : 1;
    int rc = run_inverse_workers(threads, nitems, display, [&](Worker &w, int i, int *disp) {
        const size_t b = static_cast<size_t>(i) * chunk;
        return build_inverse_pixels(w, undecided.data() + b, std::min<size_t>(chunk, undecided.size() - b), disp);
    });
    char info[160];
    snprintf(info, sizeof info, "device: %zu of %zu pixels re-evaluated by the interpreter", undecided.size(), area);
    build_info_ = info;
    return rc == 0 ? 0 : -1;
}

int FisheyeHost::build_inverse(int threads) {
    if (!fn_inverse_.is_function()) {
        print("lens_inverse is not a function\n");
        return -2;
    }
    int display[kMaxPlates] = {0, 0, 0, 0, 0, 0};
    int rc = 1;
    if (threads == 0) {
        std::string why = "no GPU lens builder installed";
        if (device_builder_) rc = build_inverse_device(display, &why);
        if (rc == 1) {
            build_info_ = "host (" + why + ")";
            threads = fallback_threads_;
        }
    }
    if (rc == 1) {
        if (threads < 1) threads = 1;
        if (build_info_.empty()) build_info_ = "host";
        const int band = threads > 1 ? 8 : height_px_;  // one thread: the reference's single bottom-up sweep
        const int nbands = (height_px_ + band - 1) / band;
        rc = run_inverse_workers(threads, nbands, display, [&](Worker &w, int b, int *disp) {
            const int y0 = b * band;
            return build_inverse_rows(w, y0, std::min(height_px_, y0 + band), disp);
        });
    }
    for (int i = 0; i < kMaxPlates; ++i) plates_[i].display = display[i];
    return rc;
}

// ---------------------------------------------------------------------------
// forward builder (fisheye.c:2126-2338)
// ---------------------------------------------------------------------------

int FisheyeHost::uv_to_screen(Worker &w, int plate, double u, double v, int *lx, int *ly) {
    float ray[3];
    plate_uv_to_ray(plate, u, v, ray);
    double x, y;
    int status = call_forward(w, ray, &x, &y);
    if (status != 1) return status;
    *lx = static_cast<int>(x / scale_ + width_px_ / 2);
    *ly = static_cast<int>(-y / scale_ + height_px_ / 2);
    return 1;
}

void FisheyeHost::draw_quad(const int *tl, const int *tr, const int *bl, const int *br, int plate, int px, int py, int *display) {
    const int *corner[4] = {tl, tr, br, bl};  // clockwise
    int x = tl[0], y = tl[1];
    int minx = x, maxx = x, miny = y, maxy = y;
    for (int i = 1; i < 4; ++i) {
        int cx = corner[i][0], cy = corner[i][1];
        if (cx < minx) minx = cx; else if (cx > maxx) maxx = cx;
        if (cy < miny) miny = cy; else if (cy > maxy) maxy = cy;
    }
    const int maxdiff = 20;  // wrap-around guard, :2271
    if (std::abs(minx - maxx) > maxdiff || std::abs(miny - maxy) > maxdiff) return;
    if (miny == maxy && minx == maxx) {
        set_from_plate(x, y, px, py, plate, display);
        return;
    }
    if (miny == maxy) {
        for (int tx = minx; tx <= maxx; ++tx) set_from_plate(tx, miny, px, py, plate, display);
        return;
    }
    if (minx == maxx) {
        for (int ty = miny; ty <= maxy; ++ty) set_from_plate(x, ty, px, py, plate, display);
        return;
    }
    for (y = miny; y <= maxy; ++y) {
        int tx[2] = {minx, maxx};
        int found = 0;
        int j = 3;
        for (int i = 0; i < 4; ++i) {
            int ix = corner[i][0], iy = corner[i][1];
            int jx = corner[j][0], jy = corner[j][1];
            if ((iy < y && y <= jy) || (jy < y && y <= iy)) {
                double dy = jy - iy;
                double dx = jx - ix;
                tx[found] = static_cast<int>(ix + (y - iy) / dy * dx);
                if (++found == 2) break;
            }
            j = i;
        }
        if (tx[0] > tx[1]) std::swap(tx[0], tx[1]);
        if (tx[1] - tx[0] > maxdiff) {
            print("%d > maxdiff\n", tx[1] - tx[0]);
            return;
        }
        for (x = tx[0]; x <= tx[1]; ++x) set_from_plate(x, y, px, py, plate, display);
    }
}

// Forward lenses on the GPU: lens_forward is evaluated at every plate grid point by the translated
// kernel, the interpreter settles the points the device could not decide, then the quads are
// rasterised on the device in the reference's writer order (lens_device.cu).
int FisheyeHost::build_forward_device(std::string *why) {
    std::string src;
    if (!lens_device_source(true, &src, why, true)) return 1;
    const LensBuildParams p = device_params();
    std::vector<uint32_t> undecided;
    if (!device_builder_->forward_points(src, p, &undecided, why)) return 1;
    std::vector<ForwardPatch> patches(undecided.size());
    const int n1 = platesize_ + 1;
    const int chunk = 256;
    const int nitems = static_cast<int>((undecided.size() + chunk - 1) / chunk);
    int display_unused[kMaxPlates] = {0, 0, 0, 0, 0, 0};
    std::atomic<int> bad(0);
    // the workers only need lens_forward; the generic worker setup parks lens_inverse (may be nil: fine)
    lua_->set_global("__blinky_forward", fn_forward_);
    int rc = run_inverse_workers(undecided.size() >= 4096 ? fallback_threads_ : 1, nitems, display_unused, [&](Worker &w, int item, int *) {
        if (!w.forward.is_function()) w.forward = w.L->get_global("__blinky_forward");
        const size_t b = static_cast<size_t>(item) * chunk, e = std::min(undecided.size(), b + chunk);
        for (size_t k = b; k < e; ++k) {
            const uint32_t pt = undecided[k];
            const int i = static_cast<int>(pt % n1), j = static_cast<int>(pt / n1 % n1), plate = static_cast<int>(pt / n1 / n1);
            ForwardPatch &out = patches[k];
            out.point = pt;
            out.lx = out.ly = 0;
            out.status = uv_to_screen(w, plate, (i - 0.5) / platesize_, (j - 0.5) / platesize_, &out.lx, &out.ly);
            if (out.status < 0) bad.store(1);
        }
        w.forward = Value();
        return 0;
    });
    lua_->set_global("__blinky_forward", Value());
    if (rc != 0 || bad.load()) return -1;
    int display[kMaxPlates] = {0, 0, 0, 0, 0, 0};
    std::vector<std::pair<uint32_t, int>> messages;
    if (!device_builder_->forward_finish(patches, idx_.data(), tint_.data(), display, &messages, why)) {
        std::fill(idx_.begin(), idx_.end(), -1);
        std::fill(tint_.begin(), tint_.end(), 255);
        return 1;
    }
    std::sort(messages.begin(), messages.end());
    for (auto &m : messages) print("%d > maxdiff\n", m.second);
    for (int i = 0; i < kMaxPlates; ++i) plates_[i].display = display[i];
    char info[160];
    snprintf(info, sizeof info, "device (forward): %zu of %zu grid points re-evaluated by the interpreter", undecided.size(),
             static_cast<size_t>(numplates_) * n1 * n1);
    build_info_ = info;
    return 0;
}

int FisheyeHost::build_forward(int threads) {
    if (!fn_forward_.is_function()) {
        print("lens_forward is not a function\n");
        return -2;
    }
    if (threads == 0) {
        std::string why = "no GPU lens builder installed";
        int rc = device_builder_ ? build_forward_device(&why) : 1;
        if (rc != 1) return rc;
        build_info_ = "host (forward lens; " + why + ")";
    }
    Worker w;
    w.L = lua_.get();
    w.forward = fn_forward_;
    w.globe_plate = fn_globe_plate_;
    w.has_globe_plate = fn_globe_plate_.is_function();
    int display[kMaxPlates] = {0, 0, 0, 0, 0, 0};
    const int ps = platesize_;
    // two rows of (ps+1) screen points; zero-initialised (the reference leaves
    // them uninitialised, which only matters if lens_forward returns nil)
    std::vector<int> rowa(static_cast<size_t>(ps + 1) * 2, 0), rowb(static_cast<size_t>(ps + 1) * 2, 0);
    int *top = rowa.data(), *bot = rowb.data();
    int rc = 0;
    try {
        for (int plate = 0; plate < numplates_ && rc == 0; ++plate) {
            for (int py = ps - 1; py >= 0 && rc == 0; --py) {
                auto fill_row = [&](int *row, double v) -> int {
                    for (int px = 0; px < ps; ++px) {
                        if (px == 0) {
                            int st = uv_to_screen(w, plate, (px - 0.5) / ps, v, &row[0], &row[1]);
                            if (st == 0) continue;
                            if (st == -1) return -1;
                        }
                        int at = 2 * (px + 1);
                        int st = uv_to_screen(w, plate, (px + 0.5) / ps, v, &row[at], &row[at + 1]);
                        if (st == 0) continue;
                        if (st == -1) return -1;
                    }
                    return 0;
                };
                if (py == ps - 1) {
                    if (fill_row(bot, (py + 0.5) / ps) != 0) { rc = -1; break; }
                } else {
                    std::swap(top, bot);  // previous top edge is this row's bottom edge
                }
                if (fill_row(top, (py - 0.5) / ps) != 0) { rc = -1; break; }
                double v = static_cast<double>(py) / ps;
                for (int px = 0; px < ps; ++px) {
                    float ray[3];
                    plate_uv_to_ray(plate, static_cast<double>(px) / ps, v, ray);
                    if (plate != ray_to_plate_index(w, ray)) continue;  // texel owned by another plate
                    int at = 2 * px;
                    draw_quad(&top[at], &top[at + 2], &bot[at], &bot[at + 2], plate, px, py, display);
                }
            }
        }
    } catch (LuaError &e) {
        print("%s\n", e.what());
        rc = -1;
    }
    for (int i = 0; i < kMaxPlates; ++i) plates_[i].display = display[i];
    return rc;
}

// ---------------------------------------------------------------------------
// the rebuild branch of F_RenderView (:730-743) + create_lensmap (:2367-2397)
// ---------------------------------------------------------------------------

bool FisheyeHost::needs_rebuild(int width, int height, int platesize) const {
    if (platesize <= 0) platesize = width < height ? width : height;
    return !built_ || width != built_w_ || height != built_h_ || platesize != built_ps_ || zoom_changed_ ||
           lens_changed_ || globe_changed_;
}

int FisheyeHost::build_lensmap(int width, int height, int platesize, int threads) {
    if (width <= 0 || height <= 0) return -1;
    if (platesize <= 0) platesize = width < height ? width : height;  // :707
    if (static_cast<int64_t>(platesize) * platesize * kMaxPlates > 0x0FFFFFFF) return -1;  // 28-bit texel index
    width_px_ = width;
    height_px_ = height;
    platesize_ = platesize;
    const size_t area = static_cast<size_t>(width) * height;
    idx_.assign(area, -1);
    tint_.assign(area, 255);
    built_ = false;
    mapped_ = 0;

    using clk = std::chrono::steady_clock;
    auto ms_since = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    auto t0 = clk::now();
    // the lens script is run again on every rebuild (:737)
    lens_valid_ = load_lens();
    if (!lens_valid_) {
        lens_name_.clear();
        print("not a valid lens\n");
    }
    lens_changed_ = globe_changed_ = zoom_changed_ = false;  // :810
    built_w_ = width;
    built_h_ = height;
    built_ps_ = platesize;
    const double ms_script = ms_since(t0);

    int rc = 0;
    double ms_zoom = 0, ms_map = 0;
    build_info_.clear();
    if (!lens_valid_ || !globe_valid_) {
        rc = -7;
    } else {
        t0 = clk::now();
        const bool zoom_ok = calc_zoom();
        ms_zoom = ms_since(t0);
        t0 = clk::now();
        if (!zoom_ok) {
            rc = -3;
        } else {
            for (int i = 0; i < numplates_; ++i) plates_[i].display = 0;
            if (map_type_ == MAP_FORWARD) {
                build_info_ = "host (forward lens)";
                rc = build_forward(threads) == 0 ? 0 : -2;
            } else if (map_type_ == MAP_INVERSE) {
                rc = build_inverse(threads) == 0 ? 0 : -2;
            } else {
                print("no inverse or forward map being used\n");
                rc = -2;
            }
        }
        ms_map = ms_since(t0);
    }
    // Whatever was mapped before a failure is still rendered by the reference;
    // publish the (possibly empty) map in every case.
    t0 = clk::now();
    finish_build();
    char t[160];
    snprintf(t, sizeof t, "; script %.1f ms, zoom %.1f ms, map %.1f ms, finish %.1f ms", ms_script, ms_zoom, ms_map, ms_since(t0));
    build_info_ += t;
    return rc;
}

void FisheyeHost::finish_build() {
    const size_t area = idx_.size();
    packed_.resize(area);
    span_off_.assign(static_cast<size_t>(height_px_) + 1, 0);
    spans_.clear();
    for (int p = 0; p < kMaxPlates; ++p) {
        plate_rect_[p][0] = plate_rect_[p][1] = platesize_;
        plate_rect_[p][2] = plate_rect_[p][3] = -1;
    }
    // rows are independent: chunks of rows in parallel, stitched together in order afterwards
    struct Part {
        std::vector<int32_t> spans;      // pairs
        std::vector<int32_t> row_count;  // spans per row
        int64_t mapped = 0;
        int rect[kMaxPlates][4];
    };
    const int rows_per = 16;
    const int nchunks = (height_px_ + rows_per - 1) / rows_per;
    std::vector<Part> parts(static_cast<size_t>(nchunks));
    const int ps = platesize_;
    const int ps2 = ps * ps;
    const bool pow2 = (ps & (ps - 1)) == 0;
    int shift = 0;
    while ((1 << shift) < ps) ++shift;
    parallel_for(nchunks, fallback_threads_, [&](int ch) {
        Part &pt = parts[static_cast<size_t>(ch)];
        for (int p = 0; p < kMaxPlates; ++p) {
            pt.rect[p][0] = pt.rect[p][1] = ps;
            pt.rect[p][2] = pt.rect[p][3] = -1;
        }
        const int y0 = ch * rows_per, y1 = std::min(height_px_, y0 + rows_per);
        for (int y = y0; y < y1; ++y) {
            int run_start = -1;
            const size_t before = pt.spans.size();
            for (int x = 0; x < width_px_; ++x) {
                const size_t at = static_cast<size_t>(y) * width_px_ + x;
                const int32_t ix = idx_[at];
                if (ix >= 0) {
                    const uint32_t t = tint_[at] == 255 ? 7u : static_cast<uint32_t>(tint_[at] & 7);
                    packed_[at] = 0x80000000u | (t << 28) | static_cast<uint32_t>(ix);
                    ++pt.mapped;
                    int plate = 0, rem = ix;
                    while (rem >= ps2) {
                        rem -= ps2;
                        ++plate;
                    }
                    int *r = pt.rect[plate < kMaxPlates ? plate : kMaxPlates - 1];
                    const int ty = pow2 ? rem >> shift : rem / ps;
                    const int tx = rem - ty * ps;
                    if (tx < r[0]) r[0] = tx;
                    if (ty < r[1]) r[1] = ty;
                    if (tx > r[2]) r[2] = tx;
                    if (ty > r[3]) r[3] = ty;
                    if (run_start < 0) run_start = x;
                } else {
                    packed_[at] = 7u << 28;
                    if (run_start >= 0) {
                        pt.spans.push_back(run_start);
                        pt.spans.push_back(x);
                        run_start = -1;
                    }
                }
            }
            if (run_start >= 0) {
                pt.spans.push_back(run_start);
                pt.spans.push_back(width_px_);
            }
            pt.row_count.push_back(static_cast<int32_t>((pt.spans.size() - before) / 2));
        }
    });
    int64_t mapped = 0;
    int row = 0;
    for (const Part &pt : parts) {
        int32_t base = static_cast<int32_t>(spans_.size() / 2);
        for (int32_t n : pt.row_count) {
            span_off_[static_cast<size_t>(row++)] = base;
            base += n;
        }
        spans_.insert(spans_.end(), pt.spans.begin(), pt.spans.end());
        mapped += pt.mapped;
        for (int p = 0; p < kMaxPlates; ++p) {
            if (pt.rect[p][0] < plate_rect_[p][0]) plate_rect_[p][0] = pt.rect[p][0];
            if (pt.rect[p][1] < plate_rect_[p][1]) plate_rect_[p][1] = pt.rect[p][1];
            if (pt.rect[p][2] > plate_rect_[p][2]) plate_rect_[p][2] = pt.rect[p][2];
            if (pt.rect[p][3] > plate_rect_[p][3]) plate_rect_[p][3] = pt.rect[p][3];
        }
    }
    span_off_[static_cast<size_t>(height_px_)] = static_cast<int32_t>(spans_.size() / 2);
    mapped_ = mapped;
    built_ = true;
}

}  // namespace blinky
