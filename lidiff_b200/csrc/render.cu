// Point-cloud rendering without a display (lidiff/vis_pcd.py's draw_geometries view, lidiff_b200/render.py): a depth-keyed splat
// of square points into a 64-bit z-buffer, then one shading pass per pixel.  The formulas and their evaluation order are stated in
// include/lidiff_b200.h; every fp64 operation is rounded on its own so that tests/render_reference.py reproduces the keys and the
// colours bit for bit.
#include "common.cuh"

#define RN_ADD __dadd_rn
#define RN_SUB __dsub_rn
#define RN_MUL __dmul_rn
#define RN_DIV __ddiv_rn

struct rv3 { double x, y, z; };

__device__ __forceinline__ double rv_dot(rv3 a, rv3 b) { return RN_ADD(RN_ADD(RN_MUL(a.x, b.x), RN_MUL(a.y, b.y)), RN_MUL(a.z, b.z)); }
__device__ __forceinline__ rv3 rv_cross(rv3 a, rv3 b) {
    return {RN_SUB(RN_MUL(a.y, b.z), RN_MUL(a.z, b.y)), RN_SUB(RN_MUL(a.z, b.x), RN_MUL(a.x, b.z)), RN_SUB(RN_MUL(a.x, b.y), RN_MUL(a.y, b.x))};
}
__device__ __forceinline__ rv3 rv_normalize(rv3 a) {
    const double l = __dsqrt_rn(rv_dot(a, a));
    return {RN_DIV(a.x, l), RN_DIV(a.y, l), RN_DIV(a.z, l)};
}
__device__ __forceinline__ rv3 rv_load(const double* v) { return {v[0], v[1], v[2]}; }

// the camera basis of the header: F = normalize(front), right = normalize(up x F), up' = normalize(F x right), eye = lookat + F d
struct RenderBasis { rv3 front, right, up, eye; };

__device__ __forceinline__ RenderBasis render_basis(const lb2_render_camera& cam) {
    RenderBasis b;
    b.front = rv_normalize(rv_load(cam.front));
    b.right = rv_normalize(rv_cross(rv_load(cam.up), b.front));
    b.up = rv_normalize(rv_cross(b.front, b.right));
    b.eye = {RN_ADD(cam.lookat[0], RN_MUL(b.front.x, cam.distance)), RN_ADD(cam.lookat[1], RN_MUL(b.front.y, cam.distance)),
             RN_ADD(cam.lookat[2], RN_MUL(b.front.z, cam.distance))};
    return b;
}

// [lo, hi) = the pixels c of an axis of `size` pixels with a <= c + 0.5 < b.  a and b are first clamped to [-1, size + 1], which
// keeps the covered pixels and the int conversion in range.  a - 0.5 may round (0 < |a| < 0.25), but never across an integer that
// changes its ceil: rounding is monotone and the integers are representable.
__device__ __forceinline__ void render_span(double centre, double half, int size, int& lo, int& hi) {
    double a = RN_SUB(centre, half), b = RN_ADD(centre, half);
    const double top = (double)size + 1.0;
    a = a < -1.0 ? -1.0 : (a > top ? top : a);
    b = b < -1.0 ? -1.0 : (b > top ? top : b);
    lo = max((int)ceil(a - 0.5), 0);
    hi = min((int)ceil(b - 0.5), size);
}

__global__ void __launch_bounds__(256) k_render_splat(const double* __restrict__ pts, int64_t n, lb2_render_camera cam, double half,
                                                      unsigned long long* __restrict__ keys) {
    __shared__ RenderBasis sb;
    if (threadIdx.x == 0) sb = render_basis(cam);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const rv3 p = {__ldg(pts + 3 * i), __ldg(pts + 3 * i + 1), __ldg(pts + 3 * i + 2)};
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;
    const RenderBasis b = sb;
    const rv3 d = {RN_SUB(p.x, b.eye.x), RN_SUB(p.y, b.eye.y), RN_SUB(p.z, b.eye.z)};
    const double depth = -rv_dot(d, b.front);
    if (!(depth > RN_MUL(1e-3, cam.distance))) return;               // the near rule (NaN depth included)
    const double u = RN_ADD(0.5 * cam.width, RN_DIV(RN_MUL(cam.focal, rv_dot(d, b.right)), depth));
    const double v = RN_SUB(0.5 * cam.height, RN_DIV(RN_MUL(cam.focal, rv_dot(d, b.up)), depth));
    if (!(u == u) || !(v == v)) return;                              // an overflowed product
    int i0, i1, j0, j1;
    render_span(u, half, cam.width, i0, i1);
    render_span(v, half, cam.height, j0, j1);
    const unsigned long long key = ((unsigned long long)__float_as_uint(__double2float_rn(depth)) << 32) | (unsigned long long)i;
    for (int j = j0; j < j1; ++j) {
        unsigned long long* row = keys + (size_t)j * cam.width;
        for (int c = i0; c < i1; ++c)
            if (key < row[c]) atomicMin(row + c, key);                  // the read only skips atomics that could not win
    }
}

// open3d's ColorMapJet: JetBase over the pieces at +-0.25 / +-0.75
__device__ __forceinline__ double jet_base(double x) {
    if (x <= -0.75) return 0.0;
    if (x <= -0.25) return RN_ADD(RN_MUL(RN_DIV(RN_SUB(x, -0.75), 0.5), 1.0), 0.0);
    if (x <= 0.25) return 1.0;
    if (x <= 0.75) return RN_ADD(RN_MUL(RN_DIV(RN_SUB(x, 0.25), 0.5), -1.0), 1.0);
    return 0.0;
}

__device__ __forceinline__ unsigned char shade_byte(float c, float factor) {
    c = __fmul_rn(c, factor);
    c = !(c > 0.0f) ? 0.0f : (c > 1.0f ? 1.0f : c);
    return (unsigned char)__float2int_rn(__fmul_rn(255.0f, c));
}

__global__ void __launch_bounds__(256) k_render_shade(const unsigned long long* __restrict__ keys, const double* __restrict__ pts,
                                                      const double* __restrict__ normals, const double* __restrict__ colors,
                                                      double z_lo, double z_hi, lb2_render_camera cam, unsigned char* __restrict__ rgb) {
    __shared__ rv3 sf;
    if (threadIdx.x == 0) sf = rv_normalize(rv_load(cam.front));
    __syncthreads();
    const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (int64_t)cam.width * cam.height) return;
    const unsigned long long key = keys[pix];
    unsigned char* out = rgb + 3 * pix;
    if (key == LB2_KEY_EMPTY) { out[0] = out[1] = out[2] = 255; return; }
    const int64_t i = (int64_t)(key & 0xFFFFFFFFull);
    float c0, c1, c2;
    if (colors) {
        c0 = __double2float_rn(__ldg(colors + 3 * i)); c1 = __double2float_rn(__ldg(colors + 3 * i + 1));
        c2 = __double2float_rn(__ldg(colors + 3 * i + 2));
    } else {
        const double z = __ldg(pts + 3 * i + 2);
        double t = z_hi == z_lo ? 0.0 : RN_DIV(RN_SUB(z, z_lo), RN_SUB(z_hi, z_lo));
        t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);                        // a height outside z_range takes the colour of its end
        const double t2 = RN_MUL(t, 2.0);
        c0 = __double2float_rn(jet_base(RN_SUB(t2, 1.5)));
        c1 = __double2float_rn(jet_base(RN_SUB(t2, 1.0)));
        c2 = __double2float_rn(jet_base(RN_SUB(t2, 0.5)));
    }
    float factor = 1.0f;
    if (normals) {
        const rv3 nv = {__ldg(normals + 3 * i), __ldg(normals + 3 * i + 1), __ldg(normals + 3 * i + 2)};
        const float dot = __double2float_rn(rv_dot(nv, sf));
        if (isfinite(dot)) factor = __fadd_rn(0.25f, __fmul_rn(0.75f, fabsf(dot)));
    }
    out[0] = shade_byte(c0, factor); out[1] = shade_byte(c1, factor); out[2] = shade_byte(c2, factor);
}

static bool render_camera_ok(const lb2_render_camera* cam) {
    return cam && cam->width > 0 && cam->height > 0 && cam->distance > 0.0 && cam->focal > 0.0;
}

extern "C" int lb2_render_splat(void* handle, void* stream, const double* pts, int64_t n, const lb2_render_camera* cam, double point_size,
                                uint64_t* keys) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && keys && render_camera_ok(cam) && n >= 0 && n < (int64_t)0xFFFFFFFFll && (pts || n == 0), "render_splat");
    LB2_REQUIRE(h, point_size > 0.0 && point_size <= 4096.0, "render_splat: point_size must be in (0, 4096]");
    if (n == 0) return LB2_OK;
    k_render_splat<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(pts, n, *cam, 0.5 * point_size, (unsigned long long*)keys);
    LB2_POST_LAUNCH(h, "k_render_splat");
    return LB2_OK;
}

extern "C" int lb2_render_shade(void* handle, void* stream, const uint64_t* keys, const double* pts, const double* normals,
                                const double* colors, double z_lo, double z_hi, const lb2_render_camera* cam, uint8_t* rgb) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && keys && rgb && render_camera_ok(cam), "render_shade");
    const int64_t npix = (int64_t)cam->width * cam->height;
    k_render_shade<<<cdiv(npix, 256), 256, 0, (cudaStream_t)stream>>>((const unsigned long long*)keys, pts, normals, colors, z_lo, z_hi,
                                                                      *cam, rgb);
    LB2_POST_LAUNCH(h, "k_render_shade");
    return LB2_OK;
}
