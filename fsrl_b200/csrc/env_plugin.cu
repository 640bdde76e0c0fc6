// A user-defined device env as a plugin of libfsrl_b200.so (fsrl_b200.envs.build_device_env, `make plugin`).
// Compiled once per env with `-include <header>`; the header includes "envs.cuh" and defines, at global scope,
// `UserEnv`: a struct with the contract of envs.cuh's built-in envs (static constexpr int D, A, S, T and the
// __device__ functions reset / observe / step), or an alias of one of them.  UserEnv becomes Env<ENV_USER>, and
// fsrl_env_plugin() returns env_table<ENV_USER>(), the launcher table a built-in kind has, built from the same
// templates: with the library's flags, a plugin of a built-in struct compiles to the same kernels as the library's.
// fsrl_env_register takes the table; the kind id is assigned there.
// A struct that also defines the optional `draw` of the drawing contract (render.cuh, DESIGN §7) gets the
// rasterizer of fsrl_env_render instantiated for it, and fsrl_env_plugin_render() returns its render_table, which
// fsrl_env_register_renderer takes; without draw nothing of the renderer is compiled and that getter returns NULL.
#include "render.cuh"

#include <type_traits>
#include <utility>

namespace fsrl {

// the template argument of this plugin's instantiations, outside the built-in kinds (the plugin's symbols are
// hidden, so plugins loaded side by side never share an instantiation)
constexpr int ENV_USER = FSRL_ENV_PLUGIN_FIRST;

// the limits every learner imposes (fsrl_env_register checks them again); build_device_env reports the text
static_assert(::UserEnv::D >= 1, "env plugin limit: D >= 1");
static_assert(::UserEnv::A >= 1 && ::UserEnv::A <= ENV_MAX_A, "env plugin limit: 1 <= A <= ENV_MAX_A (8)");
static_assert(::UserEnv::D + ::UserEnv::A <= FSRL_ENG_DX_LD, "env plugin limit: D + A <= FSRL_ENG_DX_LD (80)");
static_assert(::UserEnv::S >= 1 && ::UserEnv::S <= ENV_MAX_S, "env plugin limit: 1 <= S <= ENV_MAX_S (32)");
static_assert(::UserEnv::T >= 1, "env plugin limit: T >= 1");

template <>
struct Env<ENV_USER> : ::UserEnv {};

// The drawing contract: UserEnv may define
//   __device__ static void draw(const float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost,
//                               fsrl::render::Builder& b);
// detected by name; a draw that cannot be called so is a compile error whose text build_device_env reports.
template <typename E, typename = void>
struct has_draw : std::false_type {};
template <typename E>
struct has_draw<E, std::void_t<decltype(&E::draw)>> : std::true_type {};
template <typename E, typename = void>
struct draw_callable : std::false_type {};
template <typename E>
struct draw_callable<E, std::void_t<decltype(E::draw(std::declval<const float*>(), uint32_t{}, uint32_t{}, uint32_t{},
                                                     bool{}, std::declval<render::Builder&>()))>> : std::true_type {};
constexpr bool USER_DRAWS = has_draw<::UserEnv>::value;
static_assert(!USER_DRAWS || draw_callable<::UserEnv>::value,
              "env plugin contract: UserEnv::draw must be a __device__ static function callable as "
              "draw(const float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost, fsrl::render::Builder& b)");

// UserEnv's scene: the window [-1, 1] x [-1, 1] unless draw sets one, then at most MAX_PRIM - 1 of draw's primitives
// in order (Builder::put keeps the first MAX_PRIM), so decode's progress bar always fits.  Empty without draw, when
// nothing instantiates it.
template <typename E, bool = USER_DRAWS>
struct UserScene {
    __device__ static void draw(render::Builder&, float*, uint32_t, uint32_t, uint32_t, bool) {}
};
template <typename E>
struct UserScene<E, true> {
    __device__ static void draw(render::Builder& b, float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost) {
        b.window(0.0f, 0.0f, 1.0f, 1.0f);
        E::draw(st, seed, env, ep, cost, b);
        if (b.sc.n > render::MAX_PRIM - 1) b.sc.n = render::MAX_PRIM - 1;
    }
};

template <>
__device__ void render::scene<ENV_USER>(render::Builder& b, float* st, uint32_t seed, uint32_t env, uint32_t ep,
                                        bool cost) {
    UserScene<::UserEnv>::draw(b, st, seed, env, ep, cost);
}

// the table fsrl_env_plugin_render returns: the render launcher with draw, NULL without
template <typename E, bool = USER_DRAWS>
struct UserRenderer {
    static const fsrl_env_renderer_t* table() { return nullptr; }
};
template <typename E>
struct UserRenderer<E, true> {
    static const fsrl_env_renderer_t* table() {
        static constexpr fsrl_env_renderer_t t = render_table<ENV_USER>();
        return &t;
    }
};

}  // namespace fsrl

extern "C" __attribute__((visibility("default"))) const fsrl_env_plugin_t* fsrl_env_plugin(void) {
    static constexpr fsrl_env_plugin_t table = fsrl::env_table<fsrl::ENV_USER>();
    return &table;
}

extern "C" __attribute__((visibility("default"))) const fsrl_env_renderer_t* fsrl_env_plugin_render(void) {
    return fsrl::UserRenderer<::UserEnv>::table();
}
