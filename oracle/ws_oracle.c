/*
 * ws_oracle.c -- CPU restatement of the web-splat render hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library, and only as the checker / the reported CPU
 * baseline.  The product path (web-splat_b200/) never links or calls it.
 *
 * PARITY PINNING.  The reference (KeKsBoTer/web-splat @959a3ec) has no test
 * suite, no golden images and cannot be built here (no rustc, no Vulkan).  It
 * holds exactly one known-answer test, the radix-sort self test
 * (src/gpu_rs.rs:295-331): this oracle's sort is pinned against it
 * (tests/test_oracle.py::test_sort_kat).  Stage 1 (preprocess) and stage 3
 * (rasterise + blend) are a restatement of the reference's WGSL / Rust and are
 * "PARITY UNPINNED" by any reference artefact; they are cross-checked only by
 * an independent numpy restatement (oracle/np_oracle.py) and closed-form
 * analytic cases.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference).  Arithmetic is IEEE binary32 in the operation order written
 * here; the compiler may not contract (-ffp-contract=off), so a fused
 * multiply-add happens exactly where fmaf() is written and nowhere else.  WGSL
 * leaves operation order, contraction and the accuracy of `/` (2.5 ulp) to the
 * implementation, so this file fixes ONE conforming evaluation: dot products
 * and matrix products accumulate with fmaf(), and a quotient whose divisor is
 * shared (x/w, y/w, z/w; J's 1/z; normalize) is formed as a correctly rounded
 * reciprocal times the numerator.  The sm_90a kernels mirror it operation for
 * operation (FFMA / MUFU.RCP + Newton = __frcp_rn), which is what keeps stage 1
 * bit-exact between the two while costing ~20 % fewer instructions than the
 * round-1 "one rounding per written operation" form.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define WSO_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* f16 <-> f32.  half 2.6.0 f16::from_f32 (io/ply.rs:95-98) and WGSL           */
/* pack2x16float (preprocess.wgsl:265-267): round-to-nearest-even.            */
/* ------------------------------------------------------------------------- */
static inline uint32_t f32_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float bits_f32(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

WSO_API uint16_t wso_f32_to_f16(float f)
{
    uint32_t x = f32_bits(f);
    uint32_t sign = (x >> 16) & 0x8000u;
    uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) {                       /* inf / nan */
        if (ax > 0x7f800000u) return (uint16_t)(sign | 0x7e00u | ((ax >> 13) & 0x3ffu));
        return (uint16_t)(sign | 0x7c00u);
    }
    if (ax >= 0x477ff000u) {                       /* >= 65520 -> inf (RNE) */
        return (uint16_t)(sign | 0x7c00u);
    }
    if (ax < 0x38800000u) {                        /* subnormal half or zero (< 2^-14) */
        if (ax < 0x33000000u) return (uint16_t)sign;   /* < 2^-25 -> 0 */
        /* value = m * 2^(e-150), want round(value / 2^-24) */
        uint32_t e = ax >> 23;
        uint32_t m = (ax & 0x7fffffu) | 0x800000u;
        uint32_t shift = 126u - e;                 /* e in [102,112] -> shift in [14,24] */
        uint32_t q = m >> shift;
        uint32_t rem = m & ((1u << shift) - 1u);
        uint32_t half = 1u << (shift - 1u);
        if (rem > half || (rem == half && (q & 1u))) q++;
        return (uint16_t)(sign | q);
    }
    {
        uint32_t e = (ax >> 23) - 112u;            /* rebias 127 -> 15 */
        uint32_t m = ax & 0x7fffffu;
        uint32_t h = (e << 10) | (m >> 13);
        uint32_t rem = m & 0x1fffu;
        if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) h++;   /* carry may bump exponent: fine */
        return (uint16_t)(sign | h);
    }
}

WSO_API float wso_f16_to_f32(uint16_t h)
{
    uint32_t sign = ((uint32_t)h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1fu;
    uint32_t m = h & 0x3ffu;
    if (e == 0) {
        if (m == 0) return bits_f32(sign);
        float v = (float)m * 5.9604644775390625e-08f;   /* m * 2^-24, exact */
        return (sign ? -v : v);
    }
    if (e == 31) return bits_f32(sign | 0x7f800000u | (m << 13));
    return bits_f32(sign | ((e + 112u) << 23) | (m << 13));
}

/* ------------------------------------------------------------------------- */
/* Uniform layouts (renderer.rs:290-306, 604-619; preprocess.wgsl:26-34,77-87) */
/* ------------------------------------------------------------------------- */
typedef struct {
    float view[16];      /* column-major: m[c*4+r] */
    float view_inv[16];
    float proj[16];      /* VIEWPORT_Y_FLIP * proj (renderer.rs:328) */
    float proj_inv[16];  /* inverse of the UNflipped proj (renderer.rs:329) */
    float viewport[2];
    float focal[2];
} wso_camera_uniform;    /* 272 B */

typedef struct {
    float clip_min[4];
    float clip_max[4];
    float gaussian_scaling;
    uint32_t max_sh_deg;
    uint32_t mip_splatting;
    float kernel_size;
    float walltime;
    float scene_extend;
    uint32_t _pad[2];
    float center[4];
} wso_render_settings;   /* 80 B */

typedef struct { int32_t zero_point; float scale; uint32_t _pad[2]; } wso_quant;   /* pointcloud.rs:360-366 */
typedef struct { wso_quant color_dc, color_rest, opacity, scaling_factor; } wso_quant4; /* pointcloud.rs:389-396 */

/* camera.rs:26-35 fit_near_far; Aabb::center/radius pointcloud.rs:441-448 */
WSO_API void wso_fit_near_far(const float pos[3], const float bmin[3], const float bmax[3],
                              float *znear, float *zfar)
{
    float c[3], d2 = 0.f, r2 = 0.f;
    for (int i = 0; i < 3; i++) {
        c[i] = (bmin[i] + bmax[i]) * 0.5f;          /* midpoint: (a+b)*0.5 (cgmath Point3::midpoint) */
    }
    for (int i = 0; i < 3; i++) { float t = bmax[i] - bmin[i]; r2 = r2 + t * t; }
    float radius = sqrtf(r2) / 2.0f;
    for (int i = 0; i < 3; i++) { float t = c[i] - pos[i]; d2 = d2 + t * t; }
    float distance = sqrtf(d2);
    float zf = distance + radius;
    float zn = distance - radius;
    float lo = zf / 1000.f;
    if (!(zn > lo)) zn = lo;                        /* f32::max */
    *zfar = zf; *znear = zn;
}

/*
 * camera.rs:75-83,207-234,240-242; renderer.rs:136-141,321-343.
 * rot is (w,x,y,z) = cgmath Quaternion::new(w, xi, yj, zk); Matrix3::from(q) is
 * the world->camera rotation R.  world2view builds [[R,0],[t^T,1]], inverts and
 * transposes, i.e. view = [R | -R t] for orthonormal R; this restatement writes
 * that closed form directly in f32 (cgmath 0.18 @ff840cb, the git dependency in
 * Cargo.lock:550-552, is absent here; its general 4x4 inverse may differ from
 * the closed form in the last ulp).  view_inv = [R^T | t].
 */
WSO_API void wso_camera_uniform_build(const float pos[3], const float rot_wxyz[4],
                                      float fovx, float fovy, float znear, float zfar,
                                      uint32_t W, uint32_t H, wso_camera_uniform *u)
{
    float s = rot_wxyz[0], x = rot_wxyz[1], y = rot_wxyz[2], z = rot_wxyz[3];
    float x2 = x + x, y2 = y + y, z2 = z + z;
    float xx2 = x2 * x, xy2 = x2 * y, xz2 = x2 * z;
    float yy2 = y2 * y, yz2 = y2 * z, zz2 = z2 * z;
    float sy2 = y2 * s, sz2 = z2 * s, sx2 = x2 * s;
    /* R[c][r], cgmath Matrix3::from(Quaternion) */
    float R[3][3];
    R[0][0] = 1.f - yy2 - zz2; R[0][1] = xy2 + sz2;       R[0][2] = xz2 - sy2;
    R[1][0] = xy2 - sz2;       R[1][1] = 1.f - xx2 - zz2; R[1][2] = yz2 + sx2;
    R[2][0] = xz2 + sy2;       R[2][1] = yz2 - sx2;       R[2][2] = 1.f - xx2 - yy2;

    memset(u, 0, sizeof(*u));
    for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) {
            u->view[c * 4 + r] = R[c][r];
            u->view_inv[r * 4 + c] = R[c][r];       /* transpose */
        }
    for (int r = 0; r < 3; r++) {
        /* -(R t)_r = -((R[0][r]*tx + R[1][r]*ty) + R[2][r]*tz) */
        float acc = R[0][r] * pos[0];
        acc = acc + R[1][r] * pos[1];
        acc = acc + R[2][r] * pos[2];
        u->view[12 + r] = -acc;
        u->view_inv[12 + r] = pos[r];
    }
    u->view[15] = 1.f; u->view_inv[15] = 1.f;

    /* build_proj, camera.rs:216-234 */
    float thy = tanf(fovy / 2.f), thx = tanf(fovx / 2.f);
    float top = thy * znear, bottom = -top, right = thx * znear, left = -right;
    float p00 = 2.0f * znear / (right - left);
    float p11 = 2.0f * znear / (top - bottom);
    float p02 = (right + left) / (right - left);
    float p12 = (top + bottom) / (top - bottom);
    float p22 = zfar / (zfar - znear);
    float p23 = -(zfar * znear) / (zfar - znear);
    /* after the final transpose, column-major proj[c*4+r]: */
    float P[16]; memset(P, 0, sizeof P);
    P[0 * 4 + 0] = p00;
    P[1 * 4 + 1] = p11;
    P[2 * 4 + 0] = p02; P[2 * 4 + 1] = p12; P[2 * 4 + 2] = p22; P[2 * 4 + 3] = 1.f;
    P[3 * 4 + 2] = p23;
    /* VIEWPORT_Y_FLIP * P: negate row 1 (camera.rs:107-112, renderer.rs:328) */
    for (int c = 0; c < 4; c++)
        for (int r = 0; r < 4; r++)
            u->proj[c * 4 + r] = (r == 1) ? -P[c * 4 + r] : P[c * 4 + r];
    /* proj_inv of the unflipped matrix (unused by the hot shaders): closed form */
    u->proj_inv[0 * 4 + 0] = 1.f / p00;
    u->proj_inv[1 * 4 + 1] = 1.f / p11;
    u->proj_inv[3 * 4 + 0] = p02 / p00;  u->proj_inv[3 * 4 + 1] = p12 / p11;
    u->proj_inv[3 * 4 + 2] = 1.f;
    u->proj_inv[2 * 4 + 3] = 1.f / p23;  u->proj_inv[3 * 4 + 3] = -p22 / p23;

    u->viewport[0] = (float)W; u->viewport[1] = (float)H;
    /* fov2focal camera.rs:240-242: pixels / (2 * tan(fov*0.5)) */
    u->focal[0] = (float)W / (2.f * tanf(fovx * 0.5f));
    u->focal[1] = (float)H / (2.f * tanf(fovy * 0.5f));
}

/* ------------------------------------------------------------------------- */
/* Stage 1 -- preprocess.wgsl:163-280 / preprocess_compressed.wgsl:206-331    */
/* ------------------------------------------------------------------------- */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = { 1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                -1.0925484305920792f, 0.5462742152960396f };
static const float SH_C3[7] = { -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                -0.5900435899266435f };

typedef struct { float v[3]; } vec3;
static inline vec3 v3s(float s, vec3 a) { vec3 r = {{ s * a.v[0], s * a.v[1], s * a.v[2] }}; return r; }
static inline vec3 v3add(vec3 a, vec3 b) { vec3 r = {{ a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2] }}; return r; }
static inline vec3 v3sub(vec3 a, vec3 b) { vec3 r = {{ a.v[0] - b.v[0], a.v[1] - b.v[1], a.v[2] - b.v[2] }}; return r; }
/* acc + s * a per channel, fused */
static inline vec3 v3fma(float s, vec3 a, vec3 acc) { vec3 r = {{ fmaf(s, a.v[0], acc.v[0]), fmaf(s, a.v[1], acc.v[1]), fmaf(s, a.v[2], acc.v[2]) }}; return r; }
/* correctly rounded reciprocal (IEEE division of 1 by x) */
static inline float rcp(float x) { return 1.0f / x; }

/* evaluate_sh, preprocess.wgsl:124-154 (identical in the compressed shader :174-204).
 * sh[k] = k-th RGB coefficient triple, already decoded to f32. */
static vec3 evaluate_sh(const float dir[3], const vec3 sh[16], uint32_t deg)
{
    vec3 result = v3s(SH_C0, sh[0]);
    if (deg > 0u) {
        float x = dir[0], y = dir[1], z = dir[2];
        vec3 t = v3s((-SH_C1) * y, sh[1]);
        t = v3fma(SH_C1 * z, sh[2], t);
        t = v3fma(-(SH_C1 * x), sh[3], t);
        result = v3add(result, t);
        if (deg > 1u) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            vec3 u = v3s(SH_C2[0] * xy, sh[4]);
            u = v3fma(SH_C2[1] * yz, sh[5], u);
            u = v3fma(SH_C2[2] * (2.0f * zz - xx - yy), sh[6], u);
            u = v3fma(SH_C2[3] * xz, sh[7], u);
            u = v3fma(SH_C2[4] * (xx - yy), sh[8], u);
            result = v3add(result, u);
            if (deg > 2u) {
                vec3 w = v3s(SH_C3[0] * y * (3.0f * xx - yy), sh[9]);
                w = v3fma(SH_C3[1] * xy * z, sh[10], w);
                w = v3fma(SH_C3[2] * y * (4.0f * zz - xx - yy), sh[11], w);
                w = v3fma(SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy), sh[12], w);
                w = v3fma(SH_C3[4] * x * (4.0f * zz - xx - yy), sh[13], w);
                w = v3fma(SH_C3[5] * z * (xx - yy), sh[14], w);
                w = v3fma(SH_C3[6] * x * (xx - 3.0f * yy), sh[15], w);
                result = v3add(result, w);
            }
        }
    }
    result.v[0] = result.v[0] + 0.5f; result.v[1] = result.v[1] + 0.5f; result.v[2] = result.v[2] + 0.5f;
    return result;
}

/* mat4 (column-major) * vec4, accumulated left to right with fused multiply-adds */
static inline void m4v4(const float *m, const float v[4], float out[4])
{
    for (int r = 0; r < 4; r++) {
        float acc = m[0 * 4 + r] * v[0];
        acc = fmaf(m[1 * 4 + r], v[1], acc);
        acc = fmaf(m[2 * 4 + r], v[2], acc);
        acc = fmaf(m[3 * 4 + r], v[3], acc);
        out[r] = acc;
    }
}

typedef struct {
    int visible;
    uint16_t splat[10];  /* v1.x v1.y v2.x v2.y pos.x pos.y r g b a   (pointcloud.rs:352-358) */
    uint32_t key;
} stage1_out;

/*
 * Shared tail of both preprocess shaders, from the covariance on:
 * preprocess.wgsl:194-279 / preprocess_compressed.wgsl:244-330.
 * cov6 = (xx,xy,xz,yy,yz,zz) already multiplied by the compressed path's s2 if any.
 */
static void project_tail(const wso_camera_uniform *cam, const wso_render_settings *rs,
                         const float xyz[3], const float camspace[4], const float pos2d[4],
                         const float cov6[6], float opacity, const vec3 sh[16],
                         int compressed, stage1_out *o)
{
    const float *view = cam->view;
    float fx = cam->focal[0], fy = cam->focal[1];

    /* scale_mod, preprocess.wgsl:196-201 */
    float walltime = rs->walltime;
    float scale_mod = 0.f;
    float ddx = rs->center[0] - xyz[0], ddy = rs->center[1] - xyz[1], ddz = rs->center[2] - xyz[2];
    float dist = sqrtf(fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx)));
    float dd = 5.f * dist * rcp(rs->scene_extend);
    if (walltime > dd) {
        float t = (walltime - dd);                 /* smoothstep(0,1,t): clamp((t-0)/(1-0),0,1) */
        t = t < 0.f ? 0.f : (t > 1.f ? 1.f : t);
        scale_mod = t * t * (3.f - 2.f * t);
    }
    float scaling = rs->gaussian_scaling * scale_mod;

    /* Vrk = mat3(...) * scaling * scaling  (:204-208) : (c*s)*s per entry */
    float V[3][3];
    float c0 = cov6[0] * scaling * scaling, c1 = cov6[1] * scaling * scaling, c2 = cov6[2] * scaling * scaling;
    float c3 = cov6[3] * scaling * scaling, c4 = cov6[4] * scaling * scaling, c5 = cov6[5] * scaling * scaling;
    V[0][0] = c0; V[0][1] = c1; V[0][2] = c2;
    V[1][0] = c1; V[1][1] = c3; V[1][2] = c4;
    V[2][0] = c2; V[2][1] = c4; V[2][2] = c5;

    /* J (:209-219), as a math matrix Jm(row,col) = J_wgsl[col][row] */
    float rz = rcp(camspace[2]);                   /* 1 / z_cam, shared by the four entries */
    float rz2 = rz * rz;
    float j00 = fx * rz;
    float j20 = -(fx * camspace[0]) * rz2;
    float j11 = -(fy * rz);
    float j21 = (fy * camspace[1]) * rz2;

    /* W = transpose(mat3(view[0].xyz, view[1].xyz, view[2].xyz)) (:221): Wm(i,k) = view[i][k] */
    /* T = W * J (:222): Tm(i,0) = Wm(i,0)*j00 + Wm(i,2)*j20 ; Tm(i,1) = Wm(i,1)*j11 + Wm(i,2)*j21 */
    float T0[3], T1[3];
    for (int i = 0; i < 3; i++) {
        float w0 = view[i * 4 + 0], w1 = view[i * 4 + 1], w2 = view[i * 4 + 2];
        T0[i] = fmaf(w2, j20, w0 * j00);
        T1[i] = fmaf(w2, j21, w1 * j11);
    }
    /* cov = transpose(T) * Vrk * T (:223): A = T^T V (2x3), cov = A T (2x2) */
    float A0[3], A1[3];
    for (int j = 0; j < 3; j++) {
        float a = T0[0] * V[0][j]; a = fmaf(T0[1], V[1][j], a); a = fmaf(T0[2], V[2][j], a); A0[j] = a;
        float b = T1[0] * V[0][j]; b = fmaf(T1[1], V[1][j], b); b = fmaf(T1[2], V[2][j], b); A1[j] = b;
    }
    float cov00 = A0[0] * T0[0]; cov00 = fmaf(A0[1], T0[1], cov00); cov00 = fmaf(A0[2], T0[2], cov00);
    /* WGSL cov[0][1] = column 0, row 1 = (A row 1) . (T col 0) */
    float cov01 = A1[0] * T0[0]; cov01 = fmaf(A1[1], T0[1], cov01); cov01 = fmaf(A1[2], T0[2], cov01);
    float cov11 = A1[0] * T1[0]; cov11 = fmaf(A1[1], T1[1], cov11); cov11 = fmaf(A1[2], T1[2], cov11);

    float kernel_size = rs->kernel_size;
    if (rs->mip_splatting) {                       /* :226-236 */
        float det_0 = cov00 * cov11 - cov01 * cov01;
        det_0 = (det_0 > 1e-6f) ? det_0 : 1e-6f;   /* max(1e-6, x): NaN -> 1e-6 */
        float det_1 = (cov00 + kernel_size) * (cov11 + kernel_size) - cov01 * cov01;
        det_1 = (det_1 > 1e-6f) ? det_1 : 1e-6f;
        float coef = sqrtf(det_0 / (det_1 + 1e-6f) + 1e-6f);
        if (det_0 <= 1e-6f || det_1 <= 1e-6f) coef = 0.0f;
        opacity = opacity * coef;
    }

    float diagonal1 = cov00 + kernel_size;         /* :238-251 */
    float offDiagonal = cov01;
    float diagonal2 = cov11 + kernel_size;
    float mid = 0.5f * (diagonal1 + diagonal2);
    float hx = (diagonal1 - diagonal2) / 2.0f;
    float radius = sqrtf(fmaf(offDiagonal, offDiagonal, hx * hx));
    float lambda1, lambda2;
    if (!compressed) {
        lambda1 = mid + radius;
        float l2 = mid - radius;
        lambda2 = (l2 > 0.1f) ? l2 : 0.1f;         /* max(mid - radius, 0.1) */
    } else {                                       /* preprocess_compressed.wgsl:296-297 */
        float rr = (radius > 0.1f) ? radius : 0.1f;
        lambda1 = mid + rr;
        lambda2 = mid - rr;
    }
    float dvx = offDiagonal, dvy = lambda1 - diagonal1;
    float rdl = rcp(sqrtf(fmaf(dvy, dvy, dvx * dvx)));
    dvx = dvx * rdl; dvy = dvy * rdl;              /* normalize; (0,0) -> 0 * inf = NaN (SURVEY A.4) */
    float s1 = sqrtf(2.0f * lambda1), s2 = sqrtf(2.0f * lambda2);
    float v1x = s1 * dvx, v1y = s1 * dvy;
    float v2x = s2 * dvy, v2y = s2 * (-dvx);

    float rw = rcp(pos2d[3]);
    float vcx = pos2d[0] * rw, vcy = pos2d[1] * rw;

    /* :255-260 */
    float cpx = cam->view_inv[12], cpy = cam->view_inv[13], cpz = cam->view_inv[14];
    float dx = xyz[0] - cpx, dy = xyz[1] - cpy, dz = xyz[2] - cpz;
    float rlen = rcp(sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx))));
    float dir[3] = { dx * rlen, dy * rlen, dz * rlen };
    vec3 col = evaluate_sh(dir, sh, rs->max_sh_deg);
    for (int i = 0; i < 3; i++) col.v[i] = (col.v[i] > 0.f) ? col.v[i] : 0.f;   /* max(vec3(0), c): NaN -> 0 */

    float ivw = rcp(cam->viewport[0]), ivh = rcp(cam->viewport[1]);   /* per-frame constants */
    o->visible = 1;
    o->splat[0] = wso_f32_to_f16(v1x * ivw); o->splat[1] = wso_f32_to_f16(v1y * ivh);
    o->splat[2] = wso_f32_to_f16(v2x * ivw); o->splat[3] = wso_f32_to_f16(v2y * ivh);
    o->splat[4] = wso_f32_to_f16(vcx);      o->splat[5] = wso_f32_to_f16(vcy);
    o->splat[6] = wso_f32_to_f16(col.v[0]); o->splat[7] = wso_f32_to_f16(col.v[1]);
    o->splat[8] = wso_f32_to_f16(col.v[2]); o->splat[9] = wso_f32_to_f16(opacity);

    /* :270-274 / compressed :321-326 */
    float znear = -cam->proj[3 * 4 + 2] / cam->proj[2 * 4 + 2];
    float zfar = -cam->proj[3 * 4 + 2] / (cam->proj[2 * 4 + 2] - 1.f);
    if (!compressed) {
        o->key = f32_bits(zfar - pos2d[2]);
    } else {
        float kf = 16777215.f - (pos2d[2] - znear) / (zfar - znear) * 16777215.f;
        /* WGSL u32(f32): truncate toward zero, clamp to [0, 2^32-1]; NaN -> 0 */
        uint32_t k;
        if (!(kf > 0.f)) k = 0u; else if (kf >= 4294967296.f) k = 0xffffffffu; else k = (uint32_t)kf;
        o->key = k;
    }
}

/* returns 0 = culled.  cull tests: preprocess.wgsl:177-192 / compressed :223-233 */
static int cull_and_project(const wso_camera_uniform *cam, const wso_render_settings *rs,
                            const float xyz[3], int compressed, float camspace[4], float pos2d[4])
{
    for (int i = 0; i < 3; i++)
        if (xyz[i] < rs->clip_min[i] || xyz[i] > rs->clip_max[i]) return 0;
    float p[4] = { xyz[0], xyz[1], xyz[2], 1.f };
    m4v4(cam->view, p, camspace);
    m4v4(cam->proj, camspace, pos2d);
    float bounds = 1.2f * pos2d[3];
    float z = pos2d[2] * rcp(pos2d[3]);
    if (!compressed) {
        if (z <= 0.f || z >= 1.f || pos2d[0] < -bounds || pos2d[0] > bounds || pos2d[1] < -bounds || pos2d[1] > bounds)
            return 0;
    } else {
        if (z < 0.f || z > 1.f || pos2d[0] < -bounds || pos2d[0] > bounds || pos2d[1] < -bounds || pos2d[1] > bounds)
            return 0;
    }
    return 1;
}

/*
 * Raw layout.  gaussians: N x 28 B (pointcloud.rs:38-45); sh: N x 96 B = [[f16;3];16]
 * (io/mod.rs:65, preprocess.wgsl:114-121).  Outputs are compacted in GAUSSIAN INDEX
 * ORDER (the reference's atomicAdd slot order, preprocess.wgsl:262, is
 * nondeterministic; index order is the deterministic choice, SURVEY A.2 step 8).
 * out_splats: 10 halves per visible splat; out_keys: depth key; out_src: Gaussian
 * index of each slot (diagnostic).  Returns V.
 */
WSO_API uint32_t wso_preprocess_raw(const uint8_t *gaussians, const uint8_t *sh_coefs, uint32_t n,
                                    const wso_camera_uniform *cam, const wso_render_settings *rs,
                                    uint16_t *out_splats, uint32_t *out_keys, uint32_t *out_src)
{
    uint8_t *vis = (uint8_t *)malloc(n ? n : 1);
    stage1_out *tmp = (stage1_out *)malloc(sizeof(stage1_out) * (size_t)(n ? n : 1));
#pragma omp parallel for schedule(static)
    for (int64_t idx = 0; idx < (int64_t)n; idx++) {
        const uint8_t *g = gaussians + (size_t)idx * 28u;
        float xyz[3]; memcpy(xyz, g, 12);
        uint16_t hop; memcpy(&hop, g + 12, 2);
        uint16_t hc[6]; memcpy(hc, g + 16, 12);
        float camspace[4], pos2d[4];
        vis[idx] = 0;
        if (!cull_and_project(cam, rs, xyz, 0, camspace, pos2d)) continue;
        float cov6[6];
        for (int i = 0; i < 6; i++) cov6[i] = wso_f16_to_f32(hc[i]);
        vec3 sh[16];
        const uint8_t *s = sh_coefs + (size_t)idx * 96u;
        for (int k = 0; k < 16; k++)
            for (int ch = 0; ch < 3; ch++) {
                uint16_t h; memcpy(&h, s + (k * 3 + ch) * 2, 2);
                sh[k].v[ch] = wso_f16_to_f32(h);
            }
        project_tail(cam, rs, xyz, camspace, pos2d, cov6, wso_f16_to_f32(hop), sh, 0, &tmp[idx]);
        vis[idx] = 1;
    }
    uint32_t v = 0;
    for (uint32_t idx = 0; idx < n; idx++) {
        if (!vis[idx]) continue;
        if (out_splats) memcpy(out_splats + (size_t)v * 10u, tmp[idx].splat, 20);
        if (out_keys) out_keys[v] = tmp[idx].key;
        if (out_src) out_src[v] = idx;
        v++;
    }
    free(tmp); free(vis);
    return v;
}

/* preprocess_compressed.wgsl:137-143 */
static inline float dequantize(int32_t value, const wso_quant *q)
{
    return ((float)value - (float)q->zero_point) * q->scale;
}

/*
 * Compressed layout.  gaussians: N x 24 B (pointcloud.rs:14-24); covars: 12 B per
 * codebook entry; sh_coefs: i8, (file_deg+1)^2*3 bytes per entry where file_deg is
 * the degree the renderer was specialised on (MAX_SH_DEG injection,
 * renderer.rs:385-390; preprocess_compressed.wgsl:147-171).
 * sh_coef(): unpack4x8snorm(x)*127 = max(i/127,-1)*127 then dequantizef4.
 */
WSO_API uint32_t wso_preprocess_compressed(const uint8_t *gaussians, const int8_t *sh_coefs,
                                           const uint8_t *covars, const wso_quant4 *quant,
                                           uint32_t n, uint32_t file_sh_deg,
                                           const wso_camera_uniform *cam, const wso_render_settings *rs,
                                           uint16_t *out_splats, uint32_t *out_keys, uint32_t *out_src)
{
    uint8_t *vis = (uint8_t *)malloc(n ? n : 1);
    stage1_out *tmp = (stage1_out *)malloc(sizeof(stage1_out) * (size_t)(n ? n : 1));
    uint32_t ncoef = (file_sh_deg + 1u) * (file_sh_deg + 1u);
#pragma omp parallel for schedule(static)
    for (int64_t idx = 0; idx < (int64_t)n; idx++) {
        const uint8_t *g = gaussians + (size_t)idx * 24u;
        float xyz[3]; memcpy(xyz, g, 12);
        int8_t q_op = (int8_t)g[12], q_sf = (int8_t)g[13];
        uint32_t geo_idx, sh_idx; memcpy(&geo_idx, g + 16, 4); memcpy(&sh_idx, g + 20, 4);
        float camspace[4], pos2d[4];
        vis[idx] = 0;
        if (!cull_and_project(cam, rs, xyz, 1, camspace, pos2d)) continue;
        float opacity = dequantize((int32_t)q_op, &quant->opacity);
        float scaling_factor = expf(dequantize((int32_t)q_sf, &quant->scaling_factor));
        float s2 = scaling_factor * scaling_factor;
        uint16_t hc[6]; memcpy(hc, covars + (size_t)geo_idx * 12u, 12);
        float cov6[6];
        for (int i = 0; i < 6; i++) cov6[i] = wso_f16_to_f32(hc[i]) * s2;
        vec3 sh[16];
        for (int k = 0; k < 16; k++) sh[k].v[0] = sh[k].v[1] = sh[k].v[2] = 0.f;
        uint32_t use = (rs->max_sh_deg + 1u) * (rs->max_sh_deg + 1u);
        if (use > ncoef) use = ncoef;   /* reading past the entry is UB in the reference; callers keep max_sh_deg <= file deg */
        for (uint32_t k = 0; k < use; k++) {
            const wso_quant *q = (k == 0u) ? &quant->color_dc : &quant->color_rest;
            for (int ch = 0; ch < 3; ch++) {
                int8_t b = sh_coefs[(size_t)3u * ((size_t)sh_idx * ncoef + k) + (size_t)ch];
                float sn = (float)b / 127.f; if (sn < -1.f) sn = -1.f;      /* unpack4x8snorm */
                float val = sn * 127.f;
                sh[k].v[ch] = (val - (float)q->zero_point) * q->scale;      /* dequantizef4 */
            }
        }
        project_tail(cam, rs, xyz, camspace, pos2d, cov6, opacity, sh, 1, &tmp[idx]);
        vis[idx] = 1;
    }
    uint32_t v = 0;
    for (uint32_t idx = 0; idx < n; idx++) {
        if (!vis[idx]) continue;
        if (out_splats) memcpy(out_splats + (size_t)v * 10u, tmp[idx].splat, 20);
        if (out_keys) out_keys[v] = tmp[idx].key;
        if (out_src) out_src[v] = idx;
        v++;
    }
    free(tmp); free(vis);
    return v;
}

/* ------------------------------------------------------------------------- */
/* Stage 2 -- contract of radix_sort.wgsl:48-512 + gpu_rs.rs:865-884:          */
/* stable ascending sort of (u32 key, u32 payload) pairs.  LSD, 8-bit digits,  */
/* 4 passes, like the reference (gpu_rs.rs:14-20).                             */
/* ------------------------------------------------------------------------- */
WSO_API void wso_sort_pairs(uint32_t *keys, uint32_t *vals, uint32_t n)
{
    uint32_t *k2 = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(n ? n : 1));
    uint32_t *v2 = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(n ? n : 1));
    uint32_t *ka = keys, *va = vals, *kb = k2, *vb = v2;
    for (int pass = 0; pass < 4; pass++) {
        size_t hist[256]; memset(hist, 0, sizeof hist);
        int sh = pass * 8;
        for (uint32_t i = 0; i < n; i++) hist[(ka[i] >> sh) & 255u]++;
        size_t acc = 0;
        for (int b = 0; b < 256; b++) { size_t c = hist[b]; hist[b] = acc; acc += c; }
        for (uint32_t i = 0; i < n; i++) {
            size_t d = hist[(ka[i] >> sh) & 255u]++;
            kb[d] = ka[i]; vb[d] = va[i];
        }
        uint32_t *t = ka; ka = kb; kb = t; t = va; va = vb; vb = t;
    }
    /* 4 passes: result is back in keys/vals (ping-pong a->b->a->b->a, radix_sort.wgsl:482-509) */
    free(k2); free(v2);
}

/* ------------------------------------------------------------------------- */
/* Stage 3 -- gaussian.wgsl:30-66 + PREMULTIPLIED_ALPHA_BLENDING               */
/* (renderer.rs:63-67), restated per pixel (SURVEY App. A.3).                  */
/* ------------------------------------------------------------------------- */
#define WSO_CUTOFF 2.3539888583335364   /* gaussian.wgsl:2 */

typedef struct { double v1x, v1y, v2x, v2y, cx, cy; float rgba[4]; int ok; double ex, ey, pcx, pcy; } splat_dec;

static void decode_splat(const uint16_t *h, uint32_t W, uint32_t H, splat_dec *s)
{
    s->v1x = wso_f16_to_f32(h[0]); s->v1y = wso_f16_to_f32(h[1]);
    s->v2x = wso_f16_to_f32(h[2]); s->v2y = wso_f16_to_f32(h[3]);
    s->cx = wso_f16_to_f32(h[4]);  s->cy = wso_f16_to_f32(h[5]);
    for (int i = 0; i < 4; i++) s->rgba[i] = wso_f16_to_f32(h[6 + i]);
    /* pixel-space bounding box of the footprint {p.p <= 2*CUTOFF} (gaussian.wgsl:62):
     * offset_ndc = 2*[v1 v2]*p  =>  half extent = sqrt(2*CUTOFF)*W*|(v1x,v2x)| px (SURVEY A.3) */
    double r = sqrt(2.0 * WSO_CUTOFF);
    s->ex = r * (double)W * sqrt(s->v1x * s->v1x + s->v2x * s->v2x);
    s->ey = r * (double)H * sqrt(s->v1y * s->v1y + s->v2y * s->v2y);
    s->pcx = (s->cx + 1.0) * 0.5 * (double)W;
    s->pcy = (1.0 - s->cy) * 0.5 * (double)H;
    s->ok = isfinite(s->ex) && isfinite(s->ey) && isfinite(s->pcx) && isfinite(s->pcy);
}

/*
 * splats: V x 10 halves (stage-1 output); order: V sorted payloads (stage-2 output),
 * drawn in that order = ascending key = far -> near (renderer.rs:259, gaussian.wgsl:37).
 * out: W*H*4 f32, row 0 = top.  clear = initial dst (the caller's LoadOp::Clear colour).
 * a and exp() are evaluated in f64 (the ideal of the rasteriser's affine interpolation),
 * b rounded to f32, blend dst = src + dst*(1-b) in f32 per layer.  The reference's
 * per-blend rounding to the target format is hardware behaviour and is not emulated.
 * sens (optional, W*H f32): per pixel, an upper bound on how much the result could
 * change if a test `a > 2*CUTOFF` within +-1e-4 of the threshold flipped.
 */
/* rounding of one blended channel to the render target's storage format, as the ROP does after EVERY blend
 * (renderer.rs:63-67 blends in the target: Rgba8Unorm lib.rs:192-196 / measure.rs:184, Rgba16Float render.rs:154,
 * Rgba32Float video.rs:186).  rop < 0: no per-blend rounding (f32 accumulator, the parity oracle of the float
 * compositor).  Unorm8: saturate, scale by 255, round half to even (Vulkan/D3D float->UNORM conversion). */
static inline float rop_round(float x, int rop)
{
    if (rop == 0) {
        float c = (x > 0.f) ? x : 0.f;              /* NaN -> 0 */
        if (c > 1.f) c = 1.f;
        float q = nearbyintf(c * 255.f);            /* default rounding mode = RNE */
        return q / 255.f;
    }
    if (rop == 1) return wso_f16_to_f32(wso_f32_to_f16(x));
    return x;
}

static void composite_impl(const uint16_t *splats, const uint32_t *order, uint32_t V,
                           uint32_t W, uint32_t H, const float clear[4], float *out, float *sens, int rop)
{
    const uint32_t BAND = 16;
    uint32_t nb = (H + BAND - 1) / BAND;
    splat_dec *dec = (splat_dec *)malloc(sizeof(splat_dec) * (size_t)(V ? V : 1));
    int32_t *y0s = (int32_t *)malloc(sizeof(int32_t) * (size_t)(V ? V : 1));
    int32_t *y1s = (int32_t *)malloc(sizeof(int32_t) * (size_t)(V ? V : 1));
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)V; i++) {
        decode_splat(splats + (size_t)order[i] * 10u, W, H, &dec[i]);
        if (!dec[i].ok) { y0s[i] = 1; y1s[i] = 0; continue; }
        double lo = floor(dec[i].pcy - dec[i].ey - 1.5), hi = ceil(dec[i].pcy + dec[i].ey + 0.5);
        if (lo < 0) lo = 0;
        if (hi > (double)H - 1) hi = (double)H - 1;
        if (hi < lo) { y0s[i] = 1; y1s[i] = 0; } else { y0s[i] = (int32_t)lo; y1s[i] = (int32_t)hi; }
    }
    /* per-band ordered lists (counting pass + fill pass keeps draw order) */
    size_t *cnt = (size_t *)calloc((size_t)nb + 1, sizeof(size_t));
    for (uint32_t i = 0; i < V; i++)
        if (y1s[i] >= y0s[i])
            for (uint32_t b = (uint32_t)y0s[i] / BAND; b <= (uint32_t)y1s[i] / BAND; b++) cnt[b + 1]++;
    for (uint32_t b = 0; b < nb; b++) cnt[b + 1] += cnt[b];
    uint32_t *list = (uint32_t *)malloc(sizeof(uint32_t) * (cnt[nb] ? cnt[nb] : 1));
    size_t *fill = (size_t *)malloc(sizeof(size_t) * ((size_t)nb + 1));
    memcpy(fill, cnt, sizeof(size_t) * ((size_t)nb + 1));
    for (uint32_t i = 0; i < V; i++)
        if (y1s[i] >= y0s[i])
            for (uint32_t b = (uint32_t)y0s[i] / BAND; b <= (uint32_t)y1s[i] / BAND; b++) list[fill[b]++] = i;

    const double thr = 2.0 * WSO_CUTOFF;
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t b = 0; b < (int64_t)nb; b++) {
        uint32_t ry0 = (uint32_t)b * BAND, ry1 = ry0 + BAND; if (ry1 > H) ry1 = H;
        for (uint32_t y = ry0; y < ry1; y++)
            for (uint32_t x = 0; x < W; x++) {
                float *d = out + ((size_t)y * W + x) * 4u;
                d[0] = rop_round(clear[0], rop); d[1] = rop_round(clear[1], rop); d[2] = rop_round(clear[2], rop); d[3] = rop_round(clear[3], rop);
                if (sens) sens[(size_t)y * W + x] = 0.f;
            }
        for (size_t li = cnt[b]; li < cnt[b + 1]; li++) {
            const splat_dec *s = &dec[list[li]];
            double lo = floor(s->pcx - s->ex - 1.5), hi = ceil(s->pcx + s->ex + 0.5);
            if (lo < 0) lo = 0;
            if (hi > (double)W - 1) hi = (double)W - 1;
            if (hi < lo) continue;
            uint32_t x0 = (uint32_t)lo, x1 = (uint32_t)hi;
            uint32_t yy0 = (uint32_t)y0s[list[li]], yy1 = (uint32_t)y1s[list[li]];
            if (yy0 < ry0) yy0 = ry0;
            if (yy1 > ry1 - 1) yy1 = ry1 - 1;
            /* M = 2*[v1 v2] (columns), gaussian.wgsl:52 */
            double m00 = 2.0 * s->v1x, m10 = 2.0 * s->v1y, m01 = 2.0 * s->v2x, m11 = 2.0 * s->v2y;
            double det = m00 * m11 - m01 * m10;
            if (det == 0.0 || !isfinite(det)) continue;     /* degenerate quad: zero area */
            double i00 = m11 / det, i01 = -m01 / det, i10 = -m10 / det, i11 = m00 / det;
            for (uint32_t y = yy0; y <= yy1; y++) {
                double ndy = 1.0 - ((double)y + 0.5) / (double)H * 2.0;
                double ddy = ndy - s->cy;
                for (uint32_t x = x0; x <= x1; x++) {
                    double ndx = ((double)x + 0.5) / (double)W * 2.0 - 1.0;
                    double ddx = ndx - s->cx;
                    double p0 = i00 * ddx + i01 * ddy, p1 = i10 * ddx + i11 * ddy;
                    /* inside the quad |p| <= CUTOFF per axis (vs_main :47-50), implied by a <= 2*CUTOFF */
                    double a = p0 * p0 + p1 * p1;
                    if (sens && fabs(a - thr) < 1e-4) {
                        float m = 1.f;
                        for (int c = 0; c < 3; c++) if (s->rgba[c] > m) m = s->rgba[c];
                        sens[(size_t)y * W + x] += (float)(exp(-thr) * fabs((double)s->rgba[3])) * m;
                    }
                    if (a > thr) continue;                   /* fs_main :62 discard */
                    double bd = exp(-a) * (double)s->rgba[3];
                    if (bd > 0.99) bd = 0.99;                /* min(0.99, .) :65 */
                    float bb = (float)bd;
                    float *d = out + ((size_t)y * W + x) * 4u;
                    float om = 1.f - bb;
                    d[0] = rop_round(s->rgba[0] * bb + d[0] * om, rop);      /* src + dst*(1-src.a), renderer.rs:63-67 */
                    d[1] = rop_round(s->rgba[1] * bb + d[1] * om, rop);
                    d[2] = rop_round(s->rgba[2] * bb + d[2] * om, rop);
                    d[3] = rop_round(bb + d[3] * om, rop);
                }
            }
        }
    }
    free(fill); free(list); free(cnt); free(y1s); free(y0s); free(dec);
}

WSO_API void wso_composite(const uint16_t *splats, const uint32_t *order, uint32_t V,
                           uint32_t W, uint32_t H, const float clear[4], float *out, float *sens)
{
    composite_impl(splats, order, V, W, H, clear, out, sens, -1);
}

/*
 * ROP-faithful variant: identical walk, but the destination holds what the reference's render target would hold --
 * every blend result is rounded to the target format (format: 0 = Rgba8Unorm, 1 = Rgba16Float, 2 = Rgba32Float)
 * before the next layer reads it back.  The blend arithmetic itself is f32 (the fixed-function blender's internal
 * precision is not specified by Vulkan; f32 + one rounding to the target is the common hardware behaviour).
 * out: W*H*4 f32 holding the quantised values.  Used to MEASURE how far a float compositor (this repo's CUDA
 * path, or wso_composite) is from the reference's own target contents (tests/test_oracle.py, DESIGN.md section 5).
 */
WSO_API void wso_composite_rop(const uint16_t *splats, const uint32_t *order, uint32_t V,
                               uint32_t W, uint32_t H, const float clear[4], int format, float *out)
{
    composite_impl(splats, order, V, W, H, clear, out, NULL, format);
}

/* ------------------------------------------------------------------------- */
/* New-design intermediate (NOT in the reference): the conservative 16x16-tile */
/* rectangle of a stored splat, restated so tests can cross-check the pair     */
/* count P.  Must match web-splat_b200/csrc (DESIGN.md "tile rect").           */
/* rect = {x0,y0,x1,y1} inclusive tile coords; empty => x1 < x0.               */
/* ------------------------------------------------------------------------- */
WSO_API void wso_tile_rects(const uint16_t *splats, uint32_t V, uint32_t W, uint32_t H,
                            int32_t *rects, uint64_t *total_pairs)
{
    const float R = 2.1697876f;                    /* f32(sqrt(2*CUTOFF)) */
    int32_t tx = (int32_t)((W + 15u) / 16u), ty = (int32_t)((H + 15u) / 16u);
    uint64_t tot = 0;
    for (uint32_t i = 0; i < V; i++) {
        const uint16_t *h = splats + (size_t)i * 10u;
        float v1x = wso_f16_to_f32(h[0]), v1y = wso_f16_to_f32(h[1]);
        float v2x = wso_f16_to_f32(h[2]), v2y = wso_f16_to_f32(h[3]);
        float cx = wso_f16_to_f32(h[4]), cy = wso_f16_to_f32(h[5]);
        float fw = (float)W, fh = (float)H;
        float ex = R * (fw * sqrtf(v1x * v1x + v2x * v2x));
        float ey = R * (fh * sqrtf(v1y * v1y + v2y * v2y));
        float pcx = (cx + 1.f) * 0.5f * fw;
        float pcy = (1.f - cy) * 0.5f * fh;
        const float pad = 0.05f;
        float fx0 = floorf((pcx - ex - 0.5f - pad) * 0.0625f), fx1 = floorf((pcx + ex - 0.5f + pad) * 0.0625f);
        float fy0 = floorf((pcy - ey - 0.5f - pad) * 0.0625f), fy1 = floorf((pcy + ey - 0.5f + pad) * 0.0625f);
        int32_t *r = rects + (size_t)i * 4u;
        if (!(fx0 == fx0) || !(fx1 == fx1) || !(fy0 == fy0) || !(fy1 == fy1)) { r[0] = r[1] = 0; r[2] = r[3] = -1; continue; }
        float lx = fx0 < 0.f ? 0.f : fx0, ly = fy0 < 0.f ? 0.f : fy0;
        float hx = fx1 > (float)(tx - 1) ? (float)(tx - 1) : fx1, hy = fy1 > (float)(ty - 1) ? (float)(ty - 1) : fy1;
        if (hx < lx || hy < ly) { r[0] = r[1] = 0; r[2] = r[3] = -1; continue; }
        r[0] = (int32_t)lx; r[1] = (int32_t)ly; r[2] = (int32_t)hx; r[3] = (int32_t)hy;
        tot += (uint64_t)(r[2] - r[0] + 1) * (uint64_t)(r[3] - r[1] + 1);
    }
    if (total_pairs) *total_pairs = tot;
}

/* ------------------------------------------------------------------------------------
 * .ply vertex conversion (SURVEY.md section 8(f) N1) -- PlyReader::read_line, io/ply.rs:50-100, with
 * sigmoid (utils.rs:206-212), build_cov (utils.rs:194-203) and cgmath 0.18 (git dependency, absent from
 * /root/reference; restated from its published source): Quaternion::normalize = q * (1/|q|),
 * Matrix3::from(Quaternion) with the x2/y2/z2 doubling form, column-major Matrix3 products.
 * `vertices` is the file's binary vertex block, already in host byte order, `stride_floats` floats per
 * vertex in the fixed order x y z nx ny nz f_dc[3] f_rest[3][C-1] opacity scale[3] rot[4].
 * Outputs: n x 28 B Gaussian records, n x 96 B [[f16;3];16] SH.  Also the GenericGaussianPointCloud::new
 * statistics (io/mod.rs:63-105,185-284) exactly as the reference computes them -- f32, file order:
 * bbox[6] (grown from the zero box), center[3], up[3]; returns 1 when `up` is Some. */
static float wso_sigmoid(float x)
{
    if (x >= 0.f) return 1.f / (1.f + expf(-x));
    float e = expf(x);
    return e / (1.f + e);
}

/* Quaternion::normalize then build_cov (utils.rs:194-203).  cgmath 0.18: InnerSpace::normalize = self * (1 / magnitude),
 * Quaternion dot = s*s + v.dot(v), Vector3 dot = (x*x + y*y) + z*z, Matrix3::from(Quaternion) in the doubling form. */
static void wso_build_cov(float qw, float qx, float qy, float qz, const float sc[3], float out[6])
{
    float mag = sqrtf(qw * qw + (qx * qx + qy * qy + qz * qz));
    float inv = 1.f / mag;
    qw = qw * inv; qx = qx * inv; qy = qy * inv; qz = qz * inv;
    float x2 = qx + qx, y2 = qy + qy, z2 = qz + qz;
    float xx2 = x2 * qx, xy2 = x2 * qy, xz2 = x2 * qz, yy2 = y2 * qy, yz2 = y2 * qz, zz2 = z2 * qz;
    float sy2 = y2 * qw, sz2 = z2 * qw, sx2 = x2 * qw;
    float R[3][3] = {{1.f - yy2 - zz2, xy2 + sz2, xz2 - sy2},
                     {xy2 - sz2, 1.f - xx2 - zz2, yz2 + sx2},
                     {xz2 + sy2, yz2 - sx2, 1.f - xx2 - yy2}};   /* R[column][row] */
    float L[3][3], M[3][3];
    for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) L[c][r] = R[c][r] * sc[c];   /* r * diag(s) */
    for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) { float m = L[0][r] * L[0][c]; m = m + L[1][r] * L[1][c]; m = m + L[2][r] * L[2][c]; M[c][r] = m; }
    out[0] = M[0][0]; out[1] = M[0][1]; out[2] = M[0][2]; out[3] = M[1][1]; out[4] = M[1][2]; out[5] = M[2][2];
}

/* GenericGaussianPointCloud::new / new_compressed statistics (io/mod.rs:74-89,119-134,185-284), f32 in file order.
 * xyz: n points, `stride` floats apart; box0 = 0 (Aabb::zeroed) or 1 (Aabb::unit). */
static int wso_cloud_stats(const float *xyz, uint32_t n, uint32_t stride, float box0, float bbox[6], float center[3], float up[3])
{
    for (int d = 0; d < 3; d++) { bbox[d] = -box0; bbox[3 + d] = box0; }
    float sum[3] = {0.f, 0.f, 0.f};
    for (uint32_t i = 0; i < n; i++) {
        const float *v = xyz + (size_t)i * stride;
        for (int d = 0; d < 3; d++) {
            bbox[d] = fminf(bbox[d], v[d]); bbox[3 + d] = fmaxf(bbox[3 + d], v[d]);
            sum[d] = sum[d] + v[d];
        }
    }
    float rn = 1.0f / (float)n;
    for (int d = 0; d < 3; d++) center[d] = sum[d] * rn;
    up[0] = up[1] = up[2] = 0.f;
    int has_up = 0;
    if (n >= 3) {
        float xx = 0.f, xy = 0.f, xz = 0.f, yy = 0.f, yz = 0.f, zz = 0.f;
        for (uint32_t i = 0; i < n; i++) {
            const float *v = xyz + (size_t)i * stride;
            float rx = v[0] - center[0], ry = v[1] - center[1], rz = v[2] - center[2];
            xx += rx * rx; xy += rx * ry; xz += rx * rz; yy += ry * ry; yz += ry * rz; zz += rz * rz;
        }
        float fn = (float)n;
        xx /= fn; xy /= fn; xz /= fn; yy /= fn; yz /= fn; zz /= fn;
        float w[3] = {0.f, 0.f, 0.f};
        float det[3] = {yy * zz - yz * yz, xx * zz - xz * xz, xx * yy - xy * xy};
        float ax[3][3] = {{det[0], xz * yz - xy * zz, xy * yz - xz * yy},
                          {xz * yz - xy * zz, det[1], xy * xz - yz * xx},
                          {xy * yz - xz * yy, xy * xz - yz * xx, det[2]}};
        for (int k = 0; k < 3; k++) {
            float weight = det[k] * det[k];
            if (w[0] * ax[k][0] + w[1] * ax[k][1] + w[2] * ax[k][2] < 0.f) weight = -weight;
            for (int d = 0; d < 3; d++) w[d] += ax[k][d] * weight;
        }
        float m = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        float rm = 1.f / m;
        float nr[3] = {w[0] * rm, w[1] * rm, w[2] * rm};
        if (nr[1] < 0.f) { nr[0] = -nr[0]; nr[1] = -nr[1]; nr[2] = -nr[2]; }
        if (isfinite(nr[0]) && isfinite(nr[1]) && isfinite(nr[2])) { has_up = 1; up[0] = nr[0]; up[1] = nr[1]; up[2] = nr[2]; }
    }
    {
        float dx = bbox[3] - bbox[0], dy = bbox[4] - bbox[1], dz = bbox[5] - bbox[2];
        if (sqrtf(dx * dx + dy * dy + dz * dz) / 2.f < 10.f) has_up = 0;
    }
    return has_up;
}

WSO_API int wso_ply_convert(const float *vertices, uint32_t n, uint32_t stride_floats, uint32_t sh_deg,
                            uint8_t *gaussians, uint8_t *sh_coefs, float bbox[6], float center[3], float up[3])
{
    const uint32_t ncoef = (sh_deg + 1u) * (sh_deg + 1u);
#pragma omp parallel for schedule(static)
    for (int64_t ii = 0; ii < (int64_t)n; ii++) {
        const uint32_t i = (uint32_t)ii;
        const float *v = vertices + (size_t)i * stride_floats;
        uint16_t sh[48];
        memset(sh, 0, sizeof sh);
        for (int ch = 0; ch < 3; ch++) sh[ch] = wso_f32_to_f16(v[6 + ch]);
        for (uint32_t c = 0; c + 1u < ncoef; c++)
            for (uint32_t ch = 0; ch < 3u; ch++) sh[(c + 1u) * 3u + ch] = wso_f32_to_f16(v[9u + ch * (ncoef - 1u) + c]);
        const float *t = v + 9u + (ncoef - 1u) * 3u;
        float opacity = wso_sigmoid(t[0]);
        float sc[3] = {expf(t[1]), expf(t[2]), expf(t[3])};
        float M6[6];
        wso_build_cov(t[4], t[5], t[6], t[7], sc, M6);
        uint8_t *g = gaussians + (size_t)i * 28u;
        memcpy(g, v, 12);
        uint16_t h[8] = {wso_f32_to_f16(opacity), 0, wso_f32_to_f16(M6[0]), wso_f32_to_f16(M6[1]), wso_f32_to_f16(M6[2]),
                         wso_f32_to_f16(M6[3]), wso_f32_to_f16(M6[4]), wso_f32_to_f16(M6[5])};
        memcpy(g + 12, h, 16);
        memcpy(sh_coefs + (size_t)i * 96u, sh, 96);
    }
    return wso_cloud_stats(vertices, n, stride_floats, 0.f, bbox, center, up);
}

/* .npz array post-processing (SURVEY.md section 8(f) N2) -- NpzReader::read, io/npz.rs:58-225.
 * Inputs are the stored arrays; scaling_factor / gaussian_indices / feature_indices may be NULL.
 * Outputs: n x 24 B GaussianCompressed, num_features x 3C i8 SH codebook (dc then rest),
 * num_covars x 12 B f16 covariance codebook, and the new_compressed statistics. */
WSO_API int wso_c3dgs_convert(const uint16_t *xyz_f16, const int8_t *opacity, const int8_t *scaling_factor,
                              const int32_t *gaussian_indices, const int32_t *feature_indices, uint32_t n,
                              const int8_t *scaling, const int8_t *rotation, uint32_t num_covars,
                              const int8_t *features_dc, const int8_t *features_rest, uint32_t num_features, uint32_t sh_deg,
                              float scaling_scale, int32_t scaling_zero_point, float rotation_scale, int32_t rotation_zero_point,
                              uint8_t *gaussians, int8_t *sh_out, uint8_t *covars, float bbox[6], float center[3], float up[3])
{
    const uint32_t per = (sh_deg + 1u) * (sh_deg + 1u) * 3u, rest = per - 3u;
    float *xyz = (float *)malloc((size_t)(n ? n : 1) * 12u);
    for (uint32_t i = 0; i < n; i++) {
        uint8_t *g = gaussians + (size_t)i * 24u;
        for (int d = 0; d < 3; d++) xyz[(size_t)i * 3u + d] = wso_f16_to_f32(xyz_f16[(size_t)i * 3u + d]);
        memcpy(g, xyz + (size_t)i * 3u, 12);
        g[12] = (uint8_t)opacity[i];
        g[13] = scaling_factor ? (uint8_t)scaling_factor[i] : 0;
        g[14] = g[15] = 0;
        uint32_t gi = gaussian_indices ? (uint32_t)gaussian_indices[i] : i, fi = feature_indices ? (uint32_t)feature_indices[i] : i;
        memcpy(g + 16, &gi, 4); memcpy(g + 20, &fi, 4);
    }
    for (uint32_t e = 0; e < num_features; e++) {
        int8_t *o = sh_out + (size_t)e * per;
        o[0] = features_dc[(size_t)e * 3u]; o[1] = features_dc[(size_t)e * 3u + 1]; o[2] = features_dc[(size_t)e * 3u + 2];
        for (uint32_t j = 0; j < rest; j++) o[3u + j] = features_rest[(size_t)e * rest + j];
    }
    const float szp = (float)scaling_zero_point, rzp = (float)rotation_zero_point;
    for (uint32_t i = 0; i < num_covars; i++) {
        float s[3], q[4], M6[6];
        for (int d = 0; d < 3; d++) {
            float v = ((float)scaling[(size_t)i * 3u + d] - szp) * scaling_scale;
            s[d] = scaling_factor ? fmaxf(v, 0.f) : expf(v);
        }
        if (scaling_factor) {
            float inv = 1.f / sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
            s[0] = s[0] * inv; s[1] = s[1] * inv; s[2] = s[2] * inv;
        }
        for (int d = 0; d < 4; d++) q[d] = ((float)rotation[(size_t)i * 4u + d] - rzp) * rotation_scale;
        wso_build_cov(q[0], q[1], q[2], q[3], s, M6);
        uint16_t h[6];
        for (int d = 0; d < 6; d++) h[d] = wso_f32_to_f16(M6[d]);
        memcpy(covars + (size_t)i * 12u, h, 12);
    }
    int has_up = wso_cloud_stats(xyz, n, 3, 1.f, bbox, center, up);
    free(xyz);
    return has_up;
}

WSO_API int wso_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* bench.py sets the thread count itself (torchrun exports OMP_NUM_THREADS=1 to every rank) */
WSO_API void wso_set_num_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* Output-format conversion the callers of the reference apply after read-back
 * (bin/render.rs:237: clamp(0,1)*255 as u8 truncating) is caller code, not part of the path. */
