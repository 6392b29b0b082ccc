// scene.cpp -- reads blub's scene JSON unchanged (src/scene/mod.rs:19-43, src/scene/models.rs:11-46).
// serde_json is replaced by a ~100-line recursive-descent reader: objects, arrays, strings, numbers, true/false/null.
// Key order is free (scenes/wavegenerator.json orders the fluid block differently from the others).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>

#include "blub_core.hpp"

namespace blub {
namespace {

struct JsonValue {
    enum Kind { Null, Bool, Number, String, Array, Object } kind = Null;
    double number = 0.0;
    bool boolean = false;
    std::string string;
    std::vector<JsonValue> array;
    std::vector<std::pair<std::string, JsonValue>> object;
    const JsonValue *get(const std::string &key) const {
        if (kind != Object) return nullptr;
        for (const auto &kv : object)
            if (kv.first == key) return &kv.second;
        return nullptr;
    }
};

struct JsonParser {
    const std::string &s;
    size_t i = 0;
    explicit JsonParser(const std::string &src) : s(src) {}
    [[noreturn]] void fail(const std::string &what) const { throw std::runtime_error("scene JSON: " + what + " at byte " + std::to_string(i)); }
    void ws() {
        while (i < s.size() && (s[i] == ' ' || s[i] == '\t' || s[i] == '\n' || s[i] == '\r')) ++i;
    }
    bool eat(char c) {
        ws();
        if (i < s.size() && s[i] == c) { ++i; return true; }
        return false;
    }
    void expect(char c) {
        if (!eat(c)) fail(std::string("expected '") + c + "'");
    }
    std::string parse_string() {
        expect('"');
        std::string out;
        while (i < s.size() && s[i] != '"') {
            char c = s[i++];
            if (c == '\\') {
                if (i >= s.size()) fail("bad escape");
                char e = s[i++];
                switch (e) {
                case 'n': out += '\n'; break;
                case 't': out += '\t'; break;
                case 'r': out += '\r'; break;
                case 'b': out += '\b'; break;
                case 'f': out += '\f'; break;
                case 'u': // keep BMP escapes as '?': no scene key or path needs them
                    if (i + 4 > s.size()) fail("bad \\u escape");
                    i += 4;
                    out += '?';
                    break;
                default: out += e; break; // \" \\ \/
                }
            } else {
                out += c;
            }
        }
        if (i >= s.size()) fail("unterminated string");
        ++i;
        return out;
    }
    JsonValue parse_value() {
        ws();
        if (i >= s.size()) fail("unexpected end");
        JsonValue v;
        char c = s[i];
        if (c == '{') {
            ++i;
            v.kind = JsonValue::Object;
            if (eat('}')) return v;
            do {
                ws();
                std::string key = parse_string();
                expect(':');
                v.object.emplace_back(key, parse_value());
            } while (eat(','));
            expect('}');
        } else if (c == '[') {
            ++i;
            v.kind = JsonValue::Array;
            if (eat(']')) return v;
            do {
                v.array.push_back(parse_value());
            } while (eat(','));
            expect(']');
        } else if (c == '"') {
            v.kind = JsonValue::String;
            v.string = parse_string();
        } else if (s.compare(i, 4, "true") == 0) {
            v.kind = JsonValue::Bool; v.boolean = true; i += 4;
        } else if (s.compare(i, 5, "false") == 0) {
            v.kind = JsonValue::Bool; v.boolean = false; i += 5;
        } else if (s.compare(i, 4, "null") == 0) {
            i += 4;
        } else {
            const char *start = s.c_str() + i;
            char *end = nullptr;
            v.number = std::strtod(start, &end);
            if (end == start) fail("unexpected character");
            v.kind = JsonValue::Number;
            i += (size_t)(end - start);
        }
        return v;
    }
};

const JsonValue &need(const JsonValue &obj, const char *key) {
    const JsonValue *v = obj.get(key);
    if (!v) throw std::runtime_error(std::string("scene JSON: missing field `") + key + "`");
    return *v;
}
float num_f32(const JsonValue &v, const char *what) {
    if (v.kind != JsonValue::Number) throw std::runtime_error(std::string("scene JSON: `") + what + "` is not a number");
    return (float)v.number; // serde parses into f32
}
uint32_t num_u32(const JsonValue &v, const char *what) {
    if (v.kind != JsonValue::Number || v.number < 0 || v.number > 4294967295.0 || std::floor(v.number) != v.number)
        throw std::runtime_error(std::string("scene JSON: `") + what + "` is not a u32");
    return (uint32_t)v.number;
}
void vec3(const JsonValue &obj, const char *what, float out[3]) {
    out[0] = num_f32(need(obj, "x"), what);
    out[1] = num_f32(need(obj, "y"), what);
    out[2] = num_f32(need(obj, "z"), what);
}
// optional particle tag of a fluid cube or a source (not in the reference, whose serde structs ignore unknown keys): an integer in [0, 2^32)
uint32_t tag_of(const JsonValue &obj, const char *what) {
    const JsonValue *v = obj.get("tag");
    return v ? num_u32(*v, what) : 0u;
}

} // namespace

float scene_viscosity_grid(const SceneConfig &cfg) { return cfg.viscosity / (cfg.grid_to_world_scale * cfg.grid_to_world_scale); }

SceneConfig parse_scene_file(const std::string &path) {
    std::ifstream in(path, std::ios::binary);
    if (!in) throw std::ios_base::failure("cannot open scene file " + path);
    std::stringstream ss;
    ss << in.rdbuf();
    const std::string text = ss.str();
    JsonParser parser(text);
    JsonValue root = parser.parse_value();
    parser.ws();
    if (parser.i != text.size()) parser.fail("trailing characters");
    if (root.kind != JsonValue::Object) throw std::runtime_error("scene JSON: root is not an object");

    SceneConfig cfg;
    vec3(need(root, "gravity"), "gravity", cfg.gravity);           // SceneConfig::gravity (world space)
    const JsonValue &fluid = need(root, "fluid");                   // FluidConfig, src/scene/mod.rs:26-33
    vec3(need(fluid, "world_position"), "world_position", cfg.world_position);
    cfg.grid_to_world_scale = num_f32(need(fluid, "grid_to_world_scale"), "grid_to_world_scale");
    const JsonValue &dim = need(fluid, "grid_dimension");
    cfg.grid_dimension[0] = num_u32(need(dim, "x"), "grid_dimension");
    cfg.grid_dimension[1] = num_u32(need(dim, "y"), "grid_dimension");
    cfg.grid_dimension[2] = num_u32(need(dim, "z"), "grid_dimension");
    cfg.max_num_particles = num_u32(need(fluid, "max_num_particles"), "max_num_particles");
    const JsonValue &cubes = need(fluid, "fluid_cubes");
    if (cubes.kind != JsonValue::Array) throw std::runtime_error("scene JSON: `fluid_cubes` is not an array");
    for (const JsonValue &c : cubes.array) {
        SceneBox b;
        vec3(need(c, "min"), "fluid_cubes.min", b.min);
        vec3(need(c, "max"), "fluid_cubes.max", b.max);
        b.tag = tag_of(c, "fluid_cubes.tag");
        cfg.fluid_cubes.push_back(b);
    }
    // sources and drains (not in the reference, whose serde structs ignore unknown keys): world units and m/s, both optional
    if (const JsonValue *srcs = fluid.get("sources")) {
        if (srcs->kind != JsonValue::Array) throw std::runtime_error("scene JSON: `fluid.sources` is not an array");
        for (const JsonValue &s : srcs->array) {
            SceneSource b;
            vec3(need(s, "min"), "sources.min", b.min);
            vec3(need(s, "max"), "sources.max", b.max);
            vec3(need(s, "velocity"), "sources.velocity", b.velocity);
            b.tag = tag_of(s, "sources.tag");
            cfg.sources.push_back(b);
        }
    }
    if (const JsonValue *drns = fluid.get("drains")) {
        if (drns->kind != JsonValue::Array) throw std::runtime_error("scene JSON: `fluid.drains` is not an array");
        for (const JsonValue &d : drns->array) {
            SceneBox b;
            vec3(need(d, "min"), "drains.min", b.min);
            vec3(need(d, "max"), "drains.max", b.max);
            cfg.drains.push_back(b);
        }
    }
    // kinematic viscosity (not in the reference): a number in m^2/s
    if (const JsonValue *nu = fluid.get("viscosity")) {
        if (nu->kind != JsonValue::Number) throw std::runtime_error("scene JSON: `fluid.viscosity` is not a number");
        cfg.viscosity = num_f32(*nu, "viscosity");
        if (!std::isfinite(cfg.viscosity) || cfg.viscosity < 0.0f || !std::isfinite(scene_viscosity_grid(cfg)))
            throw std::runtime_error("scene JSON: `fluid.viscosity` must be finite and not negative");
    }
    // solid load probes (not in the reference): world units, the pivot optional
    if (const JsonValue *probes = fluid.get("load_probes")) {
        if (probes->kind != JsonValue::Array) throw std::runtime_error("scene JSON: `fluid.load_probes` is not an array");
        if (probes->array.size() > (size_t)BLUB_LOAD_PROBES_MAX) throw std::runtime_error("scene JSON: `fluid.load_probes` holds more than 16 probes");
        for (const JsonValue &p : probes->array) {
            if (p.kind != JsonValue::Object) throw std::runtime_error("scene JSON: a `fluid.load_probes` entry is not an object");
            SceneLoadProbe b;
            vec3(need(p, "min"), "load_probes.min", b.min);
            vec3(need(p, "max"), "load_probes.max", b.max);
            if (const JsonValue *pivot = p.get("pivot")) {
                vec3(*pivot, "load_probes.pivot", b.pivot);
                b.has_pivot = true;
            }
            for (int k = 0; k < 3; ++k)
                if (!std::isfinite(b.min[k]) || !std::isfinite(b.max[k]) || (b.has_pivot && !std::isfinite(b.pivot[k])))
                    throw std::runtime_error("scene JSON: a `fluid.load_probes` value is out of the float range");
            cfg.load_probes.push_back(b);
        }
    }
    // floating bodies (not in the reference): world units, m/s and rad/s; checked here against the rules of set_bodies
    if (const JsonValue *bodies = fluid.get("bodies")) {
        if (bodies->kind != JsonValue::Array) throw std::runtime_error("scene JSON: `fluid.bodies` is not an array");
        for (const JsonValue &o : bodies->array) {
            if (o.kind != JsonValue::Object) throw std::runtime_error("scene JSON: a `fluid.bodies` entry is not an object");
            SceneBody b;
            const JsonValue &shape = need(o, "shape");
            if (shape.kind != JsonValue::String || (shape.string != "box" && shape.string != "sphere" && shape.string != "mesh"))
                throw std::runtime_error("scene JSON: `bodies.shape` must be \"box\", \"sphere\" or \"mesh\"");
            b.shape = shape.string == "mesh" ? 2 : shape.string == "sphere" ? 1 : 0;
            vec3(need(o, "position"), "bodies.position", b.position);
            if (b.shape == 2) { // a closed OBJ mesh: its path relative to the scene file's directory, scale in world units per model unit
                const JsonValue &model = need(o, "model");
                if (model.kind != JsonValue::String || model.string.empty()) throw std::runtime_error("scene JSON: `bodies.model` is not a path");
                const size_t slash = path.find_last_of('/');
                b.model = model.string[0] == '/' || slash == std::string::npos ? model.string : path.substr(0, slash + 1) + model.string;
                b.model_scale = num_f32(need(o, "scale"), "bodies.scale");
                for (float &h : b.half_extent) h = 0.0f;
            } else {
                const JsonValue &ext = need(o, "half_extent"); // a sphere's radius: a number, or {x, y, z} with the radius in x
                if (ext.kind == JsonValue::Number) b.half_extent[0] = b.half_extent[1] = b.half_extent[2] = num_f32(ext, "bodies.half_extent");
                else vec3(ext, "bodies.half_extent", b.half_extent);
            }
            b.relative_density = num_f32(need(o, "relative_density"), "bodies.relative_density");
            if (const JsonValue *v = o.get("rotation_angles_deg")) vec3(*v, "bodies.rotation_angles_deg", b.rotation_angles_deg);
            if (const JsonValue *v = o.get("velocity")) vec3(*v, "bodies.velocity", b.velocity);
            if (const JsonValue *v = o.get("angular_velocity")) vec3(*v, "bodies.angular_velocity", b.angular_velocity);
            cfg.bodies.push_back(b);
        }
        try {
            const std::vector<BlubBody> grid = scene_bodies_grid(cfg);
            bool mesh = false;
            for (const SceneBody &b : cfg.bodies) mesh = mesh || b.shape == 2;
            if (!mesh) make_body_set(cfg.grid_dimension, grid.data(), (uint32_t)grid.size(), false);
            else {
                if (grid.size() > (size_t)BODIES_MAX) throw std::invalid_argument("set_bodies: at most 16 bodies");
                std::vector<BlubBody> set;
                make_mesh_body_set(cfg.grid_dimension, grid.data(), scene_body_meshes(cfg), set);
            }
        } catch (const std::exception &e) {
            throw std::runtime_error(std::string("scene JSON: `fluid.bodies`: ") + e.what());
        }
    }
    if (const JsonValue *objs = root.get("static_objects")) { // #[serde(default)]
        if (objs->kind != JsonValue::Array) throw std::runtime_error("scene JSON: `static_objects` is not an array");
        for (const JsonValue &o : objs->array) { // StaticObjectConfig, src/scene/models.rs:11-19
            SceneStaticObject so;
            const JsonValue &model = need(o, "model");
            if (model.kind != JsonValue::String) throw std::runtime_error("scene JSON: `static_objects.model` is not a string");
            so.model = model.string;
            BlubRigidObject &r = so.placement;
            std::memset(&r, 0, sizeof(r));
            r.shape = 2; // triangle mesh
            vec3(need(o, "world_position"), "static_objects.world_position", r.world_position);
            r.scale = num_f32(need(o, "scale"), "static_objects.scale");
            vec3(need(o, "rotation_angles"), "static_objects.rotation_angles", r.rotation_angles_deg);
            const JsonValue *anim = o.get("animation"); // Option<RigidAnimation>, models.rs:41-46
            if (anim && anim->kind == JsonValue::Object) {
                const JsonValue *tr = anim->get("translation"); // TranslationAnimation, :28-32
                if (tr && tr->kind == JsonValue::Object) {
                    r.has_translation = 1;
                    vec3(need(*tr, "target"), "animation.translation.target", r.translation_target);
                    const JsonValue &curve = need(*tr, "curve");
                    if (curve.kind != JsonValue::String || (curve.string != "Linear" && curve.string != "SmoothStep"))
                        throw std::runtime_error("scene JSON: `animation.translation.curve` must be \"Linear\" or \"SmoothStep\"");
                    r.translation_curve = curve.string == "SmoothStep" ? 1 : 0;
                    r.translation_duration = num_f32(need(*tr, "duration"), "animation.translation.duration");
                }
                const JsonValue *rot = anim->get("rotation"); // RotationAnimation, :35-38
                if (rot && rot->kind == JsonValue::Object) {
                    r.has_rotation = 1;
                    vec3(need(*rot, "axis"), "animation.rotation.axis", r.rotation_axis);
                    r.rotation_deg_per_sec = num_f32(need(*rot, "deg_per_sec"), "animation.rotation.deg_per_sec");
                }
            }
            cfg.static_objects.push_back(so);
        }
        cfg.num_static_objects = (uint32_t)objs->array.size();
    }
    return cfg;
}

} // namespace blub
