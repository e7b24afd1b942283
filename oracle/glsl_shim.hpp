/*
 * glsl_shim.hpp -- the part of GLSL 4.50 (and GL_KHR_shader_subgroup_*) that the renderer's compute shaders use,
 * as C++17, so that shader source translated by glsl_to_cpp.py runs on the CPU dispatch by dispatch (ref_driver.cpp).
 *
 * TEST INFRASTRUCTURE ONLY.  Written from the GLSL 4.50 specification; it holds no shader code.
 *
 * Build with -ffp-contract=off -fno-fast-math (oracle/Makefile, target `ref`): every float +, -, *, / and sqrt is one
 * correctly rounded IEEE operation, in the order the shader spells it.
 *
 * Arithmetic GLSL leaves to the implementation, and the choice made here (the oracle's documented choice, gs_oracle.c):
 *   - matrix * matrix, matrix * vector: each element is a left-to-right sum, s = a0*b0; s = s + a1*b1; ...
 *   - determinant(mat2) = m[0][0]*m[1][1] - m[1][0]*m[0][1];
 *     inverse(mat2) = adjugate * (1 / det), each element one multiply;
 *   - length(v) = sqrt((x*x + y*y) + z*z);  x / y, sqrt: correctly rounded (Vulkan allows 2.5 and 3 ulp);
 *   - exp: libm expf (exp mode 0) or the oracle's shared-definition exp, gso_exp_shared (mode 1), switched by
 *     gsr_set_exp_mode like gso_set_exp_mode;
 *   - pow(x, y) = powf (the shaders only raise 2 to small integers, which every libm returns exactly);
 *   - int(float) truncates toward zero and saturates out of range, NaN -> 0 (GLSL leaves out-of-range undefined;
 *     this is the oracle's f2i_trunc and PTX's cvt.rzi.s32.f32); uint(float) likewise on [0, 2^32);
 *   - min/max/clamp on floats return the non-NaN operand (fminf/fmaxf; GLSL leaves NaN operands undefined).
 * Everything else -- operation order, literal types, conversions, control flow -- is the shader's own.
 *
 * Invocations: a workgroup with barrier() or subgroup operations runs its invocations as cooperative fibers in a fixed
 * schedule: invocation 0, 1, 2, ... each run up to its next barrier or subgroup operation, then the next round.  Subgroup
 * operations (subgroup size 32, as sort.comp's own SUBGROUP_SIZE says) must be reached by all 32 invocations of the
 * subgroup, which the scheduler checks; shared-memory atomics are then plain read-modify-writes.
 */
#ifndef GLSL_SHIM_HPP
#define GLSL_SHIM_HPP

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <ucontext.h>

extern "C" float gso_exp_shared(float x);

namespace glsl {

using uint = uint32_t;
using std::int64_t;
using std::uint64_t;

[[noreturn]] inline void fail(const char *what) {
    std::fprintf(stderr, "glsl_shim: %s\n", what);
    std::abort();
}

/* ---------------------------------------------------------------- swizzles */
template <class T, int N> struct Swz;

/* ---------------------------------------------------------------- vectors */
#define GLSL_SWIZZLE_MEMBER(T)                                                                                          \
    template <int... I> Swz<T, (int)sizeof...(I)> swizzle() { return Swz<T, (int)sizeof...(I)>{{&(&x)[I]...}}; }      \
    T &operator[](int i) { return (&x)[i]; }                                                                            \
    const T &operator[](int i) const { return (&x)[i]; }

struct uvec2;
struct ivec2;
struct vec2 {
    float x = 0, y = 0;
    vec2() = default;
    explicit vec2(float s) : x(s), y(s) {}
    vec2(float a, float b) : x(a), y(b) {}
    explicit vec2(const uvec2 &v);
    GLSL_SWIZZLE_MEMBER(float)
};
struct vec3 {
    float x = 0, y = 0, z = 0;
    vec3() = default;
    explicit vec3(float s) : x(s), y(s), z(s) {}
    vec3(float a, float b, float c) : x(a), y(b), z(c) {}
    GLSL_SWIZZLE_MEMBER(float)
};
struct vec4 {
    float x = 0, y = 0, z = 0, w = 0;
    vec4() = default;
    explicit vec4(float s) : x(s), y(s), z(s), w(s) {}
    vec4(float a, float b, float c, float d) : x(a), y(b), z(c), w(d) {}
    vec4(const vec3 &v, float d) : x(v.x), y(v.y), z(v.z), w(d) {}
    GLSL_SWIZZLE_MEMBER(float)
};
struct uvec2 {
    uint x = 0, y = 0;
    uvec2() = default;
    uvec2(uint a, uint b) : x(a), y(b) {}
    GLSL_SWIZZLE_MEMBER(uint)
};
struct uvec3 {
    uint x = 0, y = 0, z = 0;
    uvec3() = default;
    uvec3(uint a, uint b, uint c) : x(a), y(b), z(c) {}
    GLSL_SWIZZLE_MEMBER(uint)
};
struct uvec4 {
    uint x = 0, y = 0, z = 0, w = 0;
    uvec4() = default;
    uvec4(uint a, uint b, uint c, uint d) : x(a), y(b), z(c), w(d) {}
    GLSL_SWIZZLE_MEMBER(uint)
};
struct ivec2 {
    int x = 0, y = 0;
    ivec2() = default;
    ivec2(int a, int b) : x(a), y(b) {}
    explicit ivec2(const uvec2 &v) : x((int)v.x), y((int)v.y) {}
    GLSL_SWIZZLE_MEMBER(int)
};
inline vec2::vec2(const uvec2 &v) : x((float)v.x), y((float)v.y) {}

template <class T, int N> struct VecOf;
template <> struct VecOf<float, 2> { using type = vec2; };
template <> struct VecOf<float, 3> { using type = vec3; };
template <> struct VecOf<float, 4> { using type = vec4; };
template <> struct VecOf<uint, 2> { using type = uvec2; };
template <> struct VecOf<uint, 3> { using type = uvec3; };
template <> struct VecOf<uint, 4> { using type = uvec4; };
template <> struct VecOf<int, 2> { using type = ivec2; };

/* A swizzle is a view of N components: it reads as the vector and assigns through to the components. */
template <class T, int N> struct Swz {
    T *p[N];
    using V = typename VecOf<T, N>::type;
    operator V() const {
        V v;
        for (int i = 0; i < N; i++) v[i] = *p[i];
        return v;
    }
    Swz &operator=(const V &v) {
        for (int i = 0; i < N; i++) *p[i] = v[i];
        return *this;
    }
};

#define GLSL_VEC_OPS(V, N)                                                                                              \
    inline V operator+(V a, const V &b) { for (int i = 0; i < N; i++) a[i] = a[i] + b[i]; return a; }                \
    inline V operator-(V a, const V &b) { for (int i = 0; i < N; i++) a[i] = a[i] - b[i]; return a; }                \
    inline V operator*(V a, const V &b) { for (int i = 0; i < N; i++) a[i] = a[i] * b[i]; return a; }                \
    inline V operator/(V a, const V &b) { for (int i = 0; i < N; i++) a[i] = a[i] / b[i]; return a; }                \
    inline V operator+(V a, float s) { for (int i = 0; i < N; i++) a[i] = a[i] + s; return a; }                      \
    inline V operator-(V a, float s) { for (int i = 0; i < N; i++) a[i] = a[i] - s; return a; }                      \
    inline V operator*(V a, float s) { for (int i = 0; i < N; i++) a[i] = a[i] * s; return a; }                      \
    inline V operator/(V a, float s) { for (int i = 0; i < N; i++) a[i] = a[i] / s; return a; }                      \
    inline V operator+(float s, V a) { for (int i = 0; i < N; i++) a[i] = s + a[i]; return a; }                      \
    inline V operator-(float s, V a) { for (int i = 0; i < N; i++) a[i] = s - a[i]; return a; }                      \
    inline V operator*(float s, V a) { for (int i = 0; i < N; i++) a[i] = s * a[i]; return a; }                      \
    inline V operator/(float s, V a) { for (int i = 0; i < N; i++) a[i] = s / a[i]; return a; }                      \
    inline V operator-(V a) { for (int i = 0; i < N; i++) a[i] = -a[i]; return a; }                                  \
    inline V &operator+=(V &a, const V &b) { return a = a + b; }                                                       \
    inline V &operator-=(V &a, const V &b) { return a = a - b; }                                                       \
    inline V &operator*=(V &a, const V &b) { return a = a * b; }                                                       \
    inline V &operator/=(V &a, const V &b) { return a = a / b; }                                                       \
    inline V &operator+=(V &a, float s) { return a = a + s; }                                                          \
    inline V &operator-=(V &a, float s) { return a = a - s; }                                                          \
    inline V &operator*=(V &a, float s) { return a = a * s; }                                                          \
    inline V &operator/=(V &a, float s) { return a = a / s; }
GLSL_VEC_OPS(vec2, 2)
GLSL_VEC_OPS(vec3, 3)
GLSL_VEC_OPS(vec4, 4)
#undef GLSL_VEC_OPS

/* ---------------------------------------------------------------- matrices (column-major: m[column][row]) */
struct mat4 {
    vec4 c[4];
    mat4() = default;
    vec4 &operator[](int i) { return c[i]; }
    const vec4 &operator[](int i) const { return c[i]; }
};
struct mat3 {
    vec3 c[3];
    mat3() = default;
    explicit mat3(float d) { c[0].x = c[1].y = c[2].z = d; }
    mat3(float a0, float a1, float a2, float b0, float b1, float b2, float d0, float d1, float d2)
        : c{vec3(a0, a1, a2), vec3(b0, b1, b2), vec3(d0, d1, d2)} {}
    explicit mat3(const mat4 &m) {
        for (int i = 0; i < 3; i++) c[i] = vec3(m[i].x, m[i].y, m[i].z);
    }
    vec3 &operator[](int i) { return c[i]; }
    const vec3 &operator[](int i) const { return c[i]; }
};
struct mat2 {
    vec2 c[2];
    mat2() = default;
    mat2(float a0, float a1, float b0, float b1) : c{vec2(a0, a1), vec2(b0, b1)} {}
    explicit mat2(const mat3 &m) : c{vec2(m[0].x, m[0].y), vec2(m[1].x, m[1].y)} {}
    vec2 &operator[](int i) { return c[i]; }
    const vec2 &operator[](int i) const { return c[i]; }
};

template <class M, class V, int N> inline V mat_mul_vec(const M &m, const V &v) {
    V o;
    for (int r = 0; r < N; r++) {
        float s = m[0][r] * v[0];
        for (int k = 1; k < N; k++) s = s + m[k][r] * v[k];
        o[r] = s;
    }
    return o;
}
template <class M, int N> inline M mat_mul(const M &a, const M &b) {
    M o;
    for (int c = 0; c < N; c++)
        for (int r = 0; r < N; r++) {
            float s = a[0][r] * b[c][0];
            for (int k = 1; k < N; k++) s = s + a[k][r] * b[c][k];
            o[c][r] = s;
        }
    return o;
}
template <class M, int N> inline M mat_transpose(const M &a) {
    M o;
    for (int c = 0; c < N; c++)
        for (int r = 0; r < N; r++) o[c][r] = a[r][c];
    return o;
}
inline vec4 operator*(const mat4 &m, const vec4 &v) { return mat_mul_vec<mat4, vec4, 4>(m, v); }
inline vec3 operator*(const mat3 &m, const vec3 &v) { return mat_mul_vec<mat3, vec3, 3>(m, v); }
inline vec2 operator*(const mat2 &m, const vec2 &v) { return mat_mul_vec<mat2, vec2, 2>(m, v); }
inline mat4 operator*(const mat4 &a, const mat4 &b) { return mat_mul<mat4, 4>(a, b); }
inline mat3 operator*(const mat3 &a, const mat3 &b) { return mat_mul<mat3, 3>(a, b); }
inline mat2 operator*(const mat2 &a, const mat2 &b) { return mat_mul<mat2, 2>(a, b); }
inline mat3 transpose(const mat3 &a) { return mat_transpose<mat3, 3>(a); }
inline mat2 transpose(const mat2 &a) { return mat_transpose<mat2, 2>(a); }
inline float determinant(const mat2 &m) { return m[0][0] * m[1][1] - m[1][0] * m[0][1]; }
inline mat2 inverse(const mat2 &m) {
    const float ood = 1.0f / determinant(m);
    return mat2(m[1][1] * ood, -m[0][1] * ood, -m[1][0] * ood, m[0][0] * ood);
}

/* ---------------------------------------------------------------- scalar built-ins */
inline int g_exp_mode = 0;
inline float exp(float x) { return g_exp_mode == 1 ? gso_exp_shared(x) : expf(x); }
inline float sqrt(float x) { return sqrtf(x); }
inline float ceil(float x) { return ceilf(x); }
inline float pow(float x, float y) { return powf(x, y); }
inline float min(float a, float b) { return fminf(a, b); }
inline float max(float a, float b) { return fmaxf(a, b); }
inline float clamp(float x, float lo, float hi) { return min(max(x, lo), hi); }
inline int min(int a, int b) { return b < a ? b : a; }
inline int max(int a, int b) { return a < b ? b : a; }
inline int clamp(int x, int lo, int hi) { return min(max(x, lo), hi); }
inline uint min(uint a, uint b) { return b < a ? b : a; }
inline uint max(uint a, uint b) { return a < b ? b : a; }
inline uint clamp(uint x, uint lo, uint hi) { return min(max(x, lo), hi); }
inline float length(const vec3 &v) { return sqrtf((v.x * v.x + v.y * v.y) + v.z * v.z); }
inline float length(const vec2 &v) { return sqrtf(v.x * v.x + v.y * v.y); }
inline uint floatBitsToUint(float f) {
    uint u;
    std::memcpy(&u, &f, 4);
    return u;
}
inline int bitCount(uint v) { return __builtin_popcount(v); }

/* int(...) and uint(...) constructors (the translator spells them to_int / to_uint) */
inline int to_int(float x) {
    if (x != x) return 0;
    if (x >= 2147483648.0f) return INT32_MAX;
    if (x <= -2147483648.0f) return INT32_MIN;
    return (int)x;
}
inline int to_int(double x) { return to_int((float)x); }
inline int to_int(int x) { return x; }
inline int to_int(uint x) { return (int)x; }
inline int to_int(int64_t x) { return (int)x; }
inline int to_int(uint64_t x) { return (int)x; }
inline uint to_uint(float x) {
    if (!(x > 0.0f)) return 0;
    if (x >= 4294967296.0f) return UINT32_MAX;
    return (uint)x;
}
inline uint to_uint(int x) { return (uint)x; }
inline uint to_uint(uint x) { return x; }
inline uint to_uint(int64_t x) { return (uint)x; }
inline uint to_uint(uint64_t x) { return (uint)x; }
inline uint to_uint(unsigned long long x) { return (uint)x; }

/* ---------------------------------------------------------------- resources */
/* A storage buffer's runtime array: the driver binds memory and an element count; length() is the bound count. */
template <class T> struct Buffer {
    T *data = nullptr;
    uint64_t n = 0;
    void bind(void *p, uint64_t count) {
        data = (T *)p;
        n = count;
    }
    T &operator[](uint64_t i) {
        if (i >= n) fail("storage buffer access out of range");
        return data[i];
    }
    int length() const { return (int)n; }
};
/* A storage image of RGBA32F texels, row-major. */
struct Image2D {
    float *data = nullptr;
    int width = 0, height = 0;
};
inline void imageStore(Image2D &img, ivec2 p, vec4 v) {
    if (p.x < 0 || p.y < 0 || p.x >= img.width || p.y >= img.height) return; /* out-of-bounds stores are discarded */
    float *o = img.data + ((size_t)p.y * img.width + p.x) * 4;
    o[0] = v.x;
    o[1] = v.y;
    o[2] = v.z;
    o[3] = v.w;
}

/* ---------------------------------------------------------------- invocation state */
inline uvec3 gl_GlobalInvocationID, gl_LocalInvocationID, gl_WorkGroupID, gl_NumWorkGroups;
inline uint gl_LocalInvocationIndex = 0, gl_SubgroupID = 0, gl_SubgroupInvocationID = 0;
constexpr uint SUBGROUP_SIZE_ = 32;

template <class T> inline T atomicAdd(T &mem, T v) { /* fibers never interleave inside a statement */
    const T old = mem;
    mem = old + v;
    return old;
}
inline uint atomicAdd(uint &mem, int v) { return atomicAdd<uint>(mem, (uint)v); }

/* Cooperative workgroup scheduler. */
struct Workgroup {
    int size = 0;
    std::vector<ucontext_t> ctx;
    std::vector<std::vector<char>> stacks;
    std::vector<char> done;
    std::vector<int> arrived; /* per invocation: sync points reached */
    ucontext_t sched;
    int cur = -1;
    void (*entry)() = nullptr;
    uvec3 group, num_groups, local_size;
    /* subgroup exchange, double-buffered by sync count so that one round's reads and the next round's writes don't meet */
    uint64_t slot[2][1024];
};
inline Workgroup *g_wg = nullptr;

inline void set_ids(Workgroup &w, int i) {
    const uint lx = (uint)i % w.local_size.x, ly = ((uint)i / w.local_size.x) % w.local_size.y;
    const uint lz = (uint)i / (w.local_size.x * w.local_size.y);
    gl_LocalInvocationID = uvec3(lx, ly, lz);
    gl_WorkGroupID = w.group;
    gl_NumWorkGroups = w.num_groups;
    gl_GlobalInvocationID = uvec3(w.group.x * w.local_size.x + lx, w.group.y * w.local_size.y + ly,
                                  w.group.z * w.local_size.z + lz);
    gl_LocalInvocationIndex = (uint)i;
    gl_SubgroupID = (uint)i / SUBGROUP_SIZE_;
    gl_SubgroupInvocationID = (uint)i % SUBGROUP_SIZE_;
}

inline void fiber_entry() {
    Workgroup &w = *g_wg;
    w.entry();
    w.done[w.cur] = 1;
    /* returning switches to uc_link (the scheduler) */
}

inline void sync_point() {
    Workgroup &w = *g_wg;
    if (!w.entry) return; /* a plain per-invocation loop: nothing to wait for */
    w.arrived[w.cur]++;
    swapcontext(&w.ctx[w.cur], &w.sched);
    set_ids(w, w.cur);
}

inline void barrier() { sync_point(); }
inline void memoryBarrierShared() {}
inline void groupMemoryBarrier() {}

/* Deposit v, wait for the round, and return the 32 deposits of this invocation's subgroup. */
inline const uint64_t *subgroup_exchange(uint64_t v) {
    Workgroup &w = *g_wg;
    if (!w.entry) fail("subgroup operation outside a cooperative workgroup");
    const int me = w.cur, buf = w.arrived[me] & 1, base = me - me % (int)SUBGROUP_SIZE_;
    const int my_count = w.arrived[me];
    w.slot[buf][me] = v;
    sync_point();
    for (int i = base; i < base + (int)SUBGROUP_SIZE_ && i < w.size; i++)
        if (w.arrived[i] < my_count + 1) fail("subgroup operation not reached by the whole subgroup");
    return &w.slot[buf][base];
}
inline uint subgroupAdd(uint v) {
    const uint64_t *s = subgroup_exchange(v);
    uint r = 0;
    for (uint i = 0; i < SUBGROUP_SIZE_; i++) r += (uint)s[i];
    return r;
}
inline uint subgroupExclusiveAdd(uint v) {
    const uint64_t *s = subgroup_exchange(v);
    uint r = 0;
    for (uint i = 0; i < gl_SubgroupInvocationID; i++) r += (uint)s[i];
    return r;
}
inline bool subgroupElect() {
    subgroup_exchange(1);
    return gl_SubgroupInvocationID == 0; /* every lane is active (checked above): the lowest one */
}
inline uint subgroupBroadcast(uint v, uint lane) {
    const uint64_t *s = subgroup_exchange(v);
    return (uint)s[lane];
}

/* Run one workgroup's invocations: as fibers when `cooperative`, else one after another. */
inline void run_workgroup(void (*entry)(), uvec3 group, uvec3 num_groups, uvec3 local_size, bool cooperative) {
    static Workgroup w;
    const int size = (int)(local_size.x * local_size.y * local_size.z);
    w.group = group;
    w.num_groups = num_groups;
    w.local_size = local_size;
    w.size = size;
    g_wg = &w;
    if (!cooperative) {
        w.entry = nullptr;
        for (int i = 0; i < size; i++) {
            w.cur = i;
            set_ids(w, i);
            entry();
        }
        return;
    }
    if (size > 1024) fail("workgroup too large");
    w.entry = entry;
    w.ctx.resize(size);
    w.stacks.resize(size);
    w.done.assign(size, 0);
    w.arrived.assign(size, 0);
    for (int i = 0; i < size; i++) {
        w.stacks[i].resize(1 << 16);
        getcontext(&w.ctx[i]);
        w.ctx[i].uc_stack.ss_sp = w.stacks[i].data();
        w.ctx[i].uc_stack.ss_size = w.stacks[i].size();
        w.ctx[i].uc_link = &w.sched;
        makecontext(&w.ctx[i], fiber_entry, 0);
    }
    for (;;) { /* rounds: each live invocation, in index order, runs to its next sync point */
        int ran = 0, finished = 0;
        for (int i = 0; i < size; i++) {
            if (w.done[i]) continue;
            ran++;
            w.cur = i;
            set_ids(w, i);
            swapcontext(&w.sched, &w.ctx[i]);
            finished += w.done[i];
        }
        if (!ran) break;
        if (finished && finished != ran) fail("some invocations of a workgroup returned while others wait at a barrier");
        int lo = 1 << 30, hi = -1;
        for (int i = 0; i < size; i++)
            if (!w.done[i]) {
                lo = w.arrived[i] < lo ? w.arrived[i] : lo;
                hi = w.arrived[i] > hi ? w.arrived[i] : hi;
            }
        if (hi >= 0 && lo != hi) fail("invocations of one workgroup reached different numbers of barriers");
    }
    w.entry = nullptr;
}

} // namespace glsl

#undef assert /* GLSL has none; common.glsl defines its own */

#endif
