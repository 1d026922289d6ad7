/*
 * bevy_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE)
 *
 * A plain-C restatement of the reference's per-frame visibility pipeline
 * (bevyengine/bevy 0.20.0-dev): propagate -> cull -> cluster.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this file's shared object; the product path (bevy_b200/csrc) never
 * links, calls or falls back to it.
 *
 * PINNING STATUS
 *   The reference is 100% Rust and cannot be built here (no rustc/cargo), and
 *   its arithmetic lives in the third-party crate glam = "0.33.2"
 *   (crates/bevy_math/Cargo.toml:13), which is not vendored in
 *   the reference checkout.  This file restates glam's published x86-64/SSE2
 *   operation order (see each helper) and is pinned against every golden
 *   vector the reference's own tests hold for this path:
 *     - frustum/sphere known answers    crates/bevy_camera/src/primitives.rs:462-611
 *     - obb identity equivalence        crates/bevy_camera/src/primitives.rs:802-857
 *     - contains_aabb with a real projection  primitives.rs:712-799
 *     - TRS chain propagation           crates/bevy_transform/src/helper.rs:98-146
 *     - translation-only propagation    crates/bevy_transform/src/systems.rs:855-1096
 *     - ViewVisibility 5-frame lifecycle crates/bevy_camera/src/visibility/mod.rs:1314-1448
 *     - cluster grid tiling invariants  crates/bevy_light/src/cluster/test.rs:5-54
 *     - sphere vs OBB known answers      crates/bevy_camera/src/primitives.rs:614-685 (also pins the
 *       pre-test of the SURVEY 8(f) N3 shadow-view culling at the end of this file)
 *   N3's CubemapFrusta derivation (update_point_light_frusta -> Transform::look_to -> glam
 *   Quat::from_rotation_axes) has no reference vector: "parity unpinned" for the frusta VALUES; the
 *   culling that consumes them is pinned through intersects_obb / Sphere::intersects_obb above and
 *   cross-checked against a plain loop (tests/test_oracle_next.py).
 *   Cluster MEMBERSHIP (which light lands in which cluster) has no reference
 *   test at all: for that part the oracle says "parity unpinned" and is
 *   cross-checked by a brute-force superset/subset test instead
 *   (tests/test_oracle_cluster.py).
 *
 * Floating point model: IEEE-754 binary32, round-to-nearest-even, NO FMA
 * contraction (build with -ffp-contract=off -fno-fast-math), SSE2 scalar math
 * (x86-64 default), matching a default x86-64 Rust build of glam (glam only
 * uses mul_add under target_feature="fma").
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

#define ORC_NO_PARENT 0xFFFFFFFFu  /* row has no ChildOf: a root or a flat entity */
#define ORC_DETACHED  0xFFFFFFFEu  /* has ChildOf, but parent lacks Transform/GlobalTransform (systems.rs:752-764) */

/* flags byte, shared with include/b200vis.h */
#define F_INHERITED_VISIBLE   0x01u
#define F_HAS_AABB            0x02u
#define F_HAS_SPHERE          0x04u
#define F_NO_FRUSTUM_CULLING  0x08u
#define F_HAS_VIS_RANGE       0x10u
#define F_NO_CPU_CULLING      0x20u
#define F_SPHERE_FROM_GT      0x40u
#define F_TRANSFORM_CHANGED   0x80u

#define VIEW_ACTIVE           0x01u
#define VIEW_NO_CPU_CULLING   0x02u

/* ------------------------------------------------------------------------ */
/* glam restatement (x86-64 SSE2 operation order)                            */
/* ------------------------------------------------------------------------ */
typedef struct { float x, y, z; } v3;
typedef struct { float x, y, z, w; } v4;
typedef struct { v3 x, y, z; } m3;          /* Mat3A: three columns */
typedef struct { m3 m; v3 t; } aff;         /* Affine3A */
typedef struct { v4 x, y, z, w; } m4;       /* Mat4: four columns */

static inline v3 V3(float x, float y, float z) { v3 r = {x, y, z}; return r; }
static inline v4 V4(float x, float y, float z, float w) { v4 r = {x, y, z, w}; return r; }
static inline v3 v3_add(v3 a, v3 b) { return V3(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline v3 v3_sub(v3 a, v3 b) { return V3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline v3 v3_mul(v3 a, v3 b) { return V3(a.x * b.x, a.y * b.y, a.z * b.z); }
static inline v3 v3_scale(v3 a, float s) { return V3(a.x * s, a.y * s, a.z * s); }
static inline v3 v3_neg(v3 a) { return V3(-a.x, -a.y, -a.z); }
static inline v3 v3_abs(v3 a) { return V3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
/* glam dot3 (sse2 dot3_in_x / scalar Vec3::dot): (x*x' + y*y') + z*z' */
static inline float v3_dot(v3 a, v3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static inline float v3_length(v3 a) { return sqrtf(v3_dot(a, a)); }
/* glam cross: (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x) */
static inline v3 v3_cross(v3 a, v3 b) {
    return V3(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y);
}
/* glam min/max are comparison-select (SSE _mm_min_ps/_mm_max_ps semantics): the
 * second operand wins when either is NaN. */
static inline float gl_min(float a, float b) { return a < b ? a : b; }
static inline float gl_max(float a, float b) { return a > b ? a : b; }
static inline v3 v3_min(v3 a, v3 b) { return V3(gl_min(a.x, b.x), gl_min(a.y, b.y), gl_min(a.z, b.z)); }
static inline v3 v3_max(v3 a, v3 b) { return V3(gl_max(a.x, b.x), gl_max(a.y, b.y), gl_max(a.z, b.z)); }

static inline v4 v4_add(v4 a, v4 b) { return V4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
static inline v4 v4_sub(v4 a, v4 b) { return V4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
static inline v4 v4_scale(v4 a, float s) { return V4(a.x * s, a.y * s, a.z * s, a.w * s); }
/* glam sse2 dot4_in_x: (x*x' + z*z') + (y*y' + w*w')  -- pairwise, not left to right */
static inline float v4_dot(v4 a, v4 b) { return (a.x * b.x + a.z * b.z) + (a.y * b.y + a.w * b.w); }
static inline v4 v3_extend(v3 a, float w) { return V4(a.x, a.y, a.z, w); }
static inline v3 v4_xyz(v4 a) { return V3(a.x, a.y, a.z); }

/* Mat3A * Vec3A (sse2 mul_vec3a): ((X*v.x) + (Y*v.y)) + (Z*v.z) lane-wise */
static inline v3 m3_mul_v3(const m3 *m, v3 v) {
    return v3_add(v3_add(v3_scale(m->x, v.x), v3_scale(m->y, v.y)), v3_scale(m->z, v.z));
}
static inline m3 m3_mul(const m3 *a, const m3 *b) {
    m3 r; r.x = m3_mul_v3(a, b->x); r.y = m3_mul_v3(a, b->y); r.z = m3_mul_v3(a, b->z); return r;
}
/* Mat3A::from_quat (glam f32/sse2/mat3a.rs) */
static inline m3 m3_from_quat(v4 q) {
    float x2 = q.x + q.x, y2 = q.y + q.y, z2 = q.z + q.z;
    float xx = q.x * x2, xy = q.x * y2, xz = q.x * z2;
    float yy = q.y * y2, yz = q.y * z2, zz = q.z * z2;
    float wx = q.w * x2, wy = q.w * y2, wz = q.w * z2;
    m3 r;
    r.x = V3(1.0f - (yy + zz), xy + wz, xz - wy);
    r.y = V3(xy - wz, 1.0f - (xx + zz), yz + wx);
    r.z = V3(xz + wy, yz - wx, 1.0f - (xx + yy));
    return r;
}
/* Affine3A::from_scale_rotation_translation; Transform::compute_affine
 * (crates/bevy_transform/src/components/transform.rs:273-275).  trs = t.xyz q.xyzw s.xyz */
static inline aff aff_from_trs(const float *trs) {
    m3 r = m3_from_quat(V4(trs[3], trs[4], trs[5], trs[6]));
    aff a;
    a.m.x = v3_scale(r.x, trs[7]);
    a.m.y = v3_scale(r.y, trs[8]);
    a.m.z = v3_scale(r.z, trs[9]);
    a.t = V3(trs[0], trs[1], trs[2]);
    return a;
}
/* Affine3A * Affine3A: matrix3 = A.m3*B.m3; translation = A.m3*B.t + A.t
 * (GlobalTransform::mul_transform, global_transform.rs:315-317) */
static inline aff aff_mul(const aff *a, const aff *b) {
    aff r; r.m = m3_mul(&a->m, &b->m); r.t = v3_add(m3_mul_v3(&a->m, b->t), a->t); return r;
}
static inline v3 aff_transform_point(const aff *a, v3 p) { return v3_add(m3_mul_v3(&a->m, p), a->t); }
static inline aff aff_load(const float *g) {
    aff a; a.m.x = V3(g[0], g[1], g[2]); a.m.y = V3(g[3], g[4], g[5]);
    a.m.z = V3(g[6], g[7], g[8]); a.t = V3(g[9], g[10], g[11]); return a;
}
static inline void aff_store(float *g, const aff *a) {
    g[0] = a->m.x.x; g[1] = a->m.x.y; g[2] = a->m.x.z;
    g[3] = a->m.y.x; g[4] = a->m.y.y; g[5] = a->m.y.z;
    g[6] = a->m.z.x; g[7] = a->m.z.y; g[8] = a->m.z.z;
    g[9] = a->t.x;   g[10] = a->t.y;  g[11] = a->t.z;
}
/* Mat3A::inverse (glam): cross products, det = z . (x cross y), scale, transpose */
static inline m3 m3_inverse(const m3 *m) {
    v3 t0 = v3_cross(m->y, m->z), t1 = v3_cross(m->z, m->x), t2 = v3_cross(m->x, m->y);
    float det = v3_dot(m->z, t2);
    float inv = 1.0f / det;
    v3 c0 = v3_scale(t0, inv), c1 = v3_scale(t1, inv), c2 = v3_scale(t2, inv);
    m3 r; /* transpose of (c0,c1,c2) */
    r.x = V3(c0.x, c1.x, c2.x); r.y = V3(c0.y, c1.y, c2.y); r.z = V3(c0.z, c1.z, c2.z);
    return r;
}
/* Affine3A::inverse: m = m3.inverse(); t = -(m * t) */
static inline aff aff_inverse(const aff *a) {
    aff r; r.m = m3_inverse(&a->m); r.t = v3_neg(m3_mul_v3(&r.m, a->t)); return r;
}
/* Mat4::from(Affine3A) */
static inline m4 m4_from_aff(const aff *a) {
    m4 r; r.x = v3_extend(a->m.x, 0.0f); r.y = v3_extend(a->m.y, 0.0f);
    r.z = v3_extend(a->m.z, 0.0f); r.w = v3_extend(a->t, 1.0f); return r;
}
/* Mat4 * Vec4 (sse2): (((X*v.x) + (Y*v.y)) + (Z*v.z)) + (W*v.w) */
static inline v4 m4_mul_v4(const m4 *m, v4 v) {
    return v4_add(v4_add(v4_add(v4_scale(m->x, v.x), v4_scale(m->y, v.y)), v4_scale(m->z, v.z)),
                  v4_scale(m->w, v.w));
}
static inline m4 m4_mul(const m4 *a, const m4 *b) {
    m4 r; r.x = m4_mul_v4(a, b->x); r.y = m4_mul_v4(a, b->y);
    r.z = m4_mul_v4(a, b->z); r.w = m4_mul_v4(a, b->w); return r;
}
static inline v4 m4_row(const m4 *m, int i) {
    const float *x = &m->x.x, *y = &m->y.x, *z = &m->z.x, *w = &m->w.x;
    return V4(x[i], y[i], z[i], w[i]);
}
static inline m4 m4_load(const float *p) {
    m4 r; r.x = V4(p[0], p[1], p[2], p[3]); r.y = V4(p[4], p[5], p[6], p[7]);
    r.z = V4(p[8], p[9], p[10], p[11]); r.w = V4(p[12], p[13], p[14], p[15]); return r;
}
static inline void m4_store(float *p, const m4 *m) { memcpy(p, m, 16 * sizeof(float)); }
/* Mat4::inverse -- glam's general cofactor expansion (scalar statement of the
 * sse2 kernel: same products, same subtractions, one reciprocal of the
 * determinant multiplied through). */
static m4 m4_inverse(const m4 *m) {
    float m00 = m->x.x, m01 = m->x.y, m02 = m->x.z, m03 = m->x.w;
    float m10 = m->y.x, m11 = m->y.y, m12 = m->y.z, m13 = m->y.w;
    float m20 = m->z.x, m21 = m->z.y, m22 = m->z.z, m23 = m->z.w;
    float m30 = m->w.x, m31 = m->w.y, m32 = m->w.z, m33 = m->w.w;
    float coef00 = m22 * m33 - m32 * m23;
    float coef02 = m12 * m33 - m32 * m13;
    float coef03 = m12 * m23 - m22 * m13;
    float coef04 = m21 * m33 - m31 * m23;
    float coef06 = m11 * m33 - m31 * m13;
    float coef07 = m11 * m23 - m21 * m13;
    float coef08 = m21 * m32 - m31 * m22;
    float coef10 = m11 * m32 - m31 * m12;
    float coef11 = m11 * m22 - m21 * m12;
    float coef12 = m20 * m33 - m30 * m23;
    float coef14 = m10 * m33 - m30 * m13;
    float coef15 = m10 * m23 - m20 * m13;
    float coef16 = m20 * m32 - m30 * m22;
    float coef18 = m10 * m32 - m30 * m12;
    float coef19 = m10 * m22 - m20 * m12;
    float coef20 = m20 * m31 - m30 * m21;
    float coef22 = m10 * m31 - m30 * m11;
    float coef23 = m10 * m21 - m20 * m11;
    v4 fac0 = V4(coef00, coef00, coef02, coef03);
    v4 fac1 = V4(coef04, coef04, coef06, coef07);
    v4 fac2 = V4(coef08, coef08, coef10, coef11);
    v4 fac3 = V4(coef12, coef12, coef14, coef15);
    v4 fac4 = V4(coef16, coef16, coef18, coef19);
    v4 fac5 = V4(coef20, coef20, coef22, coef23);
    v4 vec0 = V4(m10, m00, m00, m00);
    v4 vec1 = V4(m11, m01, m01, m01);
    v4 vec2 = V4(m12, m02, m02, m02);
    v4 vec3 = V4(m13, m03, m03, m03);
#define MULV(a, b) V4((a).x * (b).x, (a).y * (b).y, (a).z * (b).z, (a).w * (b).w)
    v4 inv0 = v4_add(v4_sub(MULV(vec1, fac0), MULV(vec2, fac1)), MULV(vec3, fac2));
    v4 inv1 = v4_add(v4_sub(MULV(vec0, fac0), MULV(vec2, fac3)), MULV(vec3, fac4));
    v4 inv2 = v4_add(v4_sub(MULV(vec0, fac1), MULV(vec1, fac3)), MULV(vec3, fac5));
    v4 inv3 = v4_add(v4_sub(MULV(vec0, fac2), MULV(vec1, fac4)), MULV(vec2, fac5));
    v4 sign_a = V4(1.0f, -1.0f, 1.0f, -1.0f), sign_b = V4(-1.0f, 1.0f, -1.0f, 1.0f);
    v4 i0 = MULV(inv0, sign_a), i1 = MULV(inv1, sign_b), i2 = MULV(inv2, sign_a), i3 = MULV(inv3, sign_b);
    v4 row0 = V4(i0.x, i1.x, i2.x, i3.x);
    float det = v4_dot(m->x, row0);
    float rcp = 1.0f / det;
    m4 r; r.x = v4_scale(i0, rcp); r.y = v4_scale(i1, rcp); r.z = v4_scale(i2, rcp); r.w = v4_scale(i3, rcp);
#undef MULV
    return r;
}

/* Rust `f32 as u32`: saturating, NaN -> 0 */
static inline uint32_t f32_as_u32(float f) {
    if (!(f > 0.0f)) return 0u;          /* NaN, negatives, -0 */
    if (f >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)f;
}

/* HalfSpace::new (crates/bevy_math/src/primitives/half_space.rs:53-57):
 * normal_d * normal_d.xyz().length_recip()   (Vec3 scalar length_recip = 1/sqrt(dot)) */
static inline v4 half_space_new(v4 nd) {
    float recip = 1.0f / v3_length(v4_xyz(nd));
    return v4_scale(nd, recip);
}

/* ------------------------------------------------------------------------ */
/* exported small helpers (used by the golden-vector tests)                  */
/* ------------------------------------------------------------------------ */
ORC_API void orc_half_space_new(const float *nd, float *out) {
    v4 r = half_space_new(V4(nd[0], nd[1], nd[2], nd[3])); memcpy(out, &r, 16);
}
ORC_API void orc_affine_from_trs(const float *trs, float *gt12) { aff a = aff_from_trs(trs); aff_store(gt12, &a); }
ORC_API void orc_affine_mul(const float *a12, const float *b12, float *out12) {
    aff a = aff_load(a12), b = aff_load(b12), r = aff_mul(&a, &b); aff_store(out12, &r);
}
ORC_API void orc_affine_inverse(const float *a12, float *out12) {
    aff a = aff_load(a12), r = aff_inverse(&a); aff_store(out12, &r);
}
ORC_API void orc_mat4_inverse(const float *m16, float *out16) { m4 m = m4_load(m16), r = m4_inverse(&m); m4_store(out16, &r); }
ORC_API void orc_mat4_mul(const float *a16, const float *b16, float *out16) {
    m4 a = m4_load(a16), b = m4_load(b16), r = m4_mul(&a, &b); m4_store(out16, &r);
}

/* Frustum::intersects_sphere (crates/bevy_camera/src/primitives.rs:255-268) */
static inline int frustum_intersects_sphere(const v4 *hs, v3 c, float radius, int intersect_far) {
    v4 center = v3_extend(c, 1.0f);
    int max = intersect_far ? 5 : 4;
    for (int i = 0; i <= max; ++i)
        if (v4_dot(hs[i], center) + radius <= 0.0f) return 0;
    return 1;
}
/* Aabb::relative_radius (primitives.rs:109-119) */
static inline float aabb_relative_radius(v3 half_extents, v3 p_normal, const m3 *m) {
    v3 d = V3(v3_dot(p_normal, m->x), v3_dot(p_normal, m->y), v3_dot(p_normal, m->z));
    return v3_dot(v3_abs(d), half_extents);
}
/* Frustum::intersects_obb (primitives.rs:272-294) */
static inline int frustum_intersects_obb(const v4 *hs, v3 center, v3 half_extents, const aff *wfl,
                                         int intersect_near, int intersect_far) {
    v4 c = v3_extend(aff_transform_point(wfl, center), 1.0f);
    for (int idx = 0; idx < 6; ++idx) {
        if ((idx == 4 && !intersect_near) || (idx == 5 && !intersect_far)) continue;
        v3 n = v4_xyz(hs[idx]);
        float rr = aabb_relative_radius(half_extents, n, &wfl->m);
        if (v4_dot(hs[idx], c) + rr <= 0.0f) return 0;
    }
    return 1;
}
ORC_API int orc_frustum_intersects_sphere(const float *planes24, const float *center3, float radius, int intersect_far) {
    v4 hs[6]; memcpy(hs, planes24, sizeof hs);
    return frustum_intersects_sphere(hs, V3(center3[0], center3[1], center3[2]), radius, intersect_far);
}
ORC_API int orc_frustum_intersects_obb(const float *planes24, const float *center3, const float *half3,
                                       const float *gt12, int intersect_near, int intersect_far) {
    v4 hs[6]; memcpy(hs, planes24, sizeof hs);
    aff a = aff_load(gt12);
    return frustum_intersects_obb(hs, V3(center3[0], center3[1], center3[2]), V3(half3[0], half3[1], half3[2]),
                                  &a, intersect_near, intersect_far);
}
/* Frustum::intersects_obb_identity (primitives.rs:298-309) */
ORC_API int orc_frustum_intersects_obb_identity(const float *planes24, const float *center3, const float *half3) {
    v4 hs[6]; memcpy(hs, planes24, sizeof hs);
    v4 c = V4(center3[0], center3[1], center3[2], 1.0f);
    v3 he = v3_abs(V3(half3[0], half3[1], half3[2]));
    for (int i = 0; i < 6; ++i) {
        float rr = v3_dot(he, v3_abs(v4_xyz(hs[i])));
        if (v4_dot(hs[i], c) + rr <= 0.0f) return 0;
    }
    return 1;
}
/* Aabb::is_in_half_space / Frustum::contains_aabb (primitives.rs:130-143, 313-320) */
ORC_API int orc_frustum_contains_aabb(const float *planes24, const float *center3, const float *half3, const float *gt12) {
    v4 hs[6]; memcpy(hs, planes24, sizeof hs);
    aff a = aff_load(gt12);
    m3 am; am.x = v3_abs(a.m.x); am.y = v3_abs(a.m.y); am.z = v3_abs(a.m.z);
    v3 hew = m3_mul_v3(&am, v3_abs(V3(half3[0], half3[1], half3[2])));
    v3 cw = aff_transform_point(&a, V3(center3[0], center3[1], center3[2]));
    for (int i = 0; i < 6; ++i) {
        v3 n = v4_xyz(hs[i]);
        float r = v3_dot(hew, v3_abs(n));
        float sd = v3_dot(n, cw) + hs[i].w;
        if (!(sd > r)) return 0;
    }
    return 1;
}
/* Sphere::intersects_obb (primitives.rs:219-226) */
ORC_API int orc_sphere_intersects_obb(const float *sc3, float sr, const float *center3, const float *half3, const float *gt12) {
    aff a = aff_load(gt12);
    v3 cw = aff_transform_point(&a, V3(center3[0], center3[1], center3[2]));
    v3 v = v3_sub(cw, V3(sc3[0], sc3[1], sc3[2]));
    float d_sq = v3_dot(v, v), d = sqrtf(d_sq);
    float rr = aabb_relative_radius(V3(half3[0], half3[1], half3[2]), v, &a.m);
    return d_sq <= sr * d + rr;
}

/* glam::camera::rh::proj::directx perspective_infinite_reverse (as used by
 * PerspectiveProjection::get_clip_from_view, crates/bevy_camera/src/projection.rs:339-343) */
ORC_API void orc_perspective_infinite_reverse_rh(float fov_y, float aspect, float z_near, float *out16) {
    float f = 1.0f / tanf(0.5f * fov_y);
    m4 r; r.x = V4(f / aspect, 0, 0, 0); r.y = V4(0, f, 0, 0); r.z = V4(0, 0, 0, -1.0f); r.w = V4(0, 0, z_near, 0);
    m4_store(out16, &r);
}
/* CameraProjection::compute_frustum (projection.rs:72-80) +
 * ViewFrustum::from_clip_from_world_custom_far (view_frustum.rs:51-62, 92-107) */
/* GlobalTransform::back (global_transform.rs): matrix3 * Vec3::Z, normalised */
static inline v3 gt_back(const aff *g) {
    v3 zt = m3_mul_v3(&g->m, V3(0.0f, 0.0f, 1.0f));   /* matrix3 * Vec3::Z */
    float len_recip = 1.0f / v3_length(zt);
    return v3_scale(zt, len_recip);
}
/* ViewFrustum::from_clip_from_world_custom_far (view_frustum.rs:51-62, 92-107) */
static inline void view_frustum_custom_far(const m4 *cfw, v3 view_translation, v3 view_backward, float far, v4 *hs) {
    v4 r0 = m4_row(cfw, 0), r1 = m4_row(cfw, 1), r2 = m4_row(cfw, 2), r3 = m4_row(cfw, 3);
    hs[0] = half_space_new(v4_add(r3, r0));
    hs[1] = half_space_new(v4_sub(r3, r0));
    hs[2] = half_space_new(v4_add(r3, r1));
    hs[3] = half_space_new(v4_sub(r3, r1));
    hs[4] = half_space_new(v4_add(r3, r2));
    /* custom far: the plane through view_translation - far * view_backward facing view_backward */
    v3 far_center = v3_sub(view_translation, v3_scale(view_backward, far));
    hs[5] = half_space_new(v3_extend(view_backward, -v3_dot(view_backward, far_center)));
}
ORC_API void orc_compute_frustum(const float *clip_from_view16, const float *camera_gt12, float far, float *planes24) {
    m4 cfv = m4_load(clip_from_view16);
    aff cam = aff_load(camera_gt12), inv = aff_inverse(&cam);
    m4 vfw = m4_from_aff(&inv);
    m4 cfw = m4_mul(&cfv, &vfw);
    v4 hs[6];
    view_frustum_custom_far(&cfw, cam.t, gt_back(&cam), far, hs);
    memcpy(planes24, hs, sizeof hs);
}

/* ------------------------------------------------------------------------ */
/* stage 1: propagate                                                        */
/* ------------------------------------------------------------------------ */
/* IEEE `!=` over the 12 floats (Affine3A: PartialEq; set_if_neq,
 * crates/bevy_ecs/src/change_detection/traits.rs:221-233) */
static inline int gt_neq(const float *a, const float *b) {
    for (int i = 0; i < 12; ++i) if (a[i] != b[i]) return 1;
    return 0;
}

/*
 * mark_dirty_trees + propagate_parent_transforms + sync_simple_transforms
 * (crates/bevy_transform/src/systems.rs:42-79, 111-306, 506-581, 679-748).
 *
 * parent[r]   : ORC_NO_PARENT | ORC_DETACHED | parent row
 * trs[r][10]  : t.xyz q.xyzw s.xyz
 * gt[r][12]   : in = last frame's GlobalTransform, out = this frame's
 * tchanged[r] : Changed<Transform> | Changed<ChildOf> | Added<GlobalTransform> | orphaned this frame
 * gt_ext_changed[r] (may be NULL): GlobalTransform changed/added since the
 *               system last ran by something else (feeds p_global_transform.is_changed())
 * static_opt  : StaticTransformOptimizations::Enabled (1) / Disabled (0)
 * changed[r]  : out, 1 where Changed<GlobalTransform> would fire
 * returns 0, or -1 on a parent index out of range, -2 on a cycle.
 */
ORC_API int orc_propagate(uint32_t n, const uint32_t *parent, const float *trs, float *gt,
                          const uint8_t *tchanged, const uint8_t *gt_ext_changed, int static_opt,
                          uint8_t *changed) {
    memset(changed, 0, n);
    if (n == 0) return 0;
    /* children CSR */
    uint32_t *first = (uint32_t *)calloc((size_t)n + 1, sizeof(uint32_t));
    uint32_t *kids = (uint32_t *)malloc((size_t)n * sizeof(uint32_t));
    uint32_t *stack = (uint32_t *)malloc((size_t)n * sizeof(uint32_t));
    uint8_t *dirty = (uint8_t *)calloc(n, 1);
    uint8_t *state = (uint8_t *)calloc(n, 1);
    int rc = 0;
    for (uint32_t r = 0; r < n; ++r) {
        uint32_t p = parent[r];
        if (p == ORC_NO_PARENT || p == ORC_DETACHED) continue;
        if (p >= n) { rc = -1; goto done; }
        first[p + 1]++;
    }
    for (uint32_t r = 0; r < n; ++r) first[r + 1] += first[r];
    {
        uint32_t *cur = (uint32_t *)malloc((size_t)n * sizeof(uint32_t));
        memcpy(cur, first, (size_t)n * sizeof(uint32_t));
        for (uint32_t r = 0; r < n; ++r) {
            uint32_t p = parent[r];
            if (p < n) kids[cur[p]++] = r;
        }
        free(cur);
    }
    /* cycle check: every chain must end at NO_PARENT / DETACHED.  state: 1 = on path, 2 = ok */
    for (uint32_t r = 0; r < n; ++r) {
        if (state[r]) continue;
        uint32_t sp = 0, c = r;
        while (1) {
            if (state[c] == 2) break;
            if (state[c] == 1) { rc = -2; goto done; }
            state[c] = 1; stack[sp++] = c;
            uint32_t p = parent[c];
            if (p >= n) break;
            c = p;
        }
        while (sp) state[stack[--sp]] = 2;
    }
    /* mark_dirty_trees (systems.rs:134-150): climb ancestors until an already dirty one */
    if (static_opt) {
        for (uint32_t r = 0; r < n; ++r) {
            if (!tchanged[r]) continue;
            uint32_t c = r;
            while (!dirty[c]) {
                dirty[c] = 1;
                uint32_t p = parent[c];
                if (p >= n) break;
                c = p;
            }
        }
    }
    for (uint32_t r = 0; r < n; ++r) {
        if (parent[r] != ORC_NO_PARENT) continue;
        int has_children = first[r + 1] > first[r];
        if (!has_children) {
            /* sync_simple_transforms (systems.rs:42-79) */
            if (tchanged[r]) {
                aff a = aff_from_trs(trs + (size_t)r * 10);
                aff_store(gt + (size_t)r * 12, &a);
                changed[r] = 1;
            }
            continue;
        }
        /* root with children (systems.rs:522-552) */
        if (static_opt && !dirty[r]) continue;
        {
            aff a = aff_from_trs(trs + (size_t)r * 10);
            aff_store(gt + (size_t)r * 12, &a);      /* unconditional write => changed */
            changed[r] = 1;
        }
        uint32_t sp = 0;
        stack[sp++] = r;
        while (sp) {
            uint32_t p = stack[--sp];
            int p_changed = changed[p] || (gt_ext_changed && gt_ext_changed[p]);
            aff pg = aff_load(gt + (size_t)p * 12);
            for (uint32_t k = first[p]; k < first[p + 1]; ++k) {
                uint32_t c = kids[k];
                /* static scene optimisation (systems.rs:708-714) */
                if (static_opt && !dirty[c] && !p_changed) continue;
                aff l = aff_from_trs(trs + (size_t)c * 10);
                aff g = aff_mul(&pg, &l);
                float tmp[12];
                aff_store(tmp, &g);
                /* set_if_neq (systems.rs:719) */
                if (gt_neq(tmp, gt + (size_t)c * 12)) {
                    memcpy(gt + (size_t)c * 12, tmp, sizeof tmp);
                    changed[c] = 1;
                }
                if (first[c + 1] > first[c]) stack[sp++] = c;
            }
        }
    }
done:
    free(first); free(kids); free(stack); free(dirty); free(state);
    return rc;
}

/* ------------------------------------------------------------------------ */
/* stage 2: cull                                                             */
/* ------------------------------------------------------------------------ */
typedef struct { uint64_t key; uint32_t row; } sort_item;
static int cmp_sort_item(const void *a, const void *b) {
    uint64_t ka = ((const sort_item *)a)->key, kb = ((const sort_item *)b)->key;
    return ka < kb ? -1 : (ka > kb ? 1 : 0);
}

/* RenderLayers is a SmallVec of 64-bit blocks (render_layers.rs:20-23); intersects() ORs the block-wise ANDs over the
 * common prefix (:121-135).  Block 0 travels in the layer_mask arguments; blocks 1..3 (layers 64..255) are registered here
 * for the next orc_cull call(s): entity_ext[n][3], view_ext[V][3], NULL = every further block empty. */
static const uint64_t *g_entity_layers_ext = NULL, *g_view_layers_ext = NULL;
static uint32_t g_current_view = 0;   /* the view orc_cull is working on (single-threaded oracle) */
ORC_API void orc_set_render_layers_ext(const uint64_t *entity_ext, const uint64_t *view_ext) {
    g_entity_layers_ext = entity_ext; g_view_layers_ext = view_ext;
}
static inline int layers_ext_intersect(uint32_t r, uint32_t v) {
    if (!g_entity_layers_ext || !g_view_layers_ext) return 0;
    for (int k = 0; k < 3; ++k)
        if (g_entity_layers_ext[(size_t)r * 3 + k] & g_view_layers_ext[(size_t)v * 3 + k]) return 1;
    return 0;
}
/* one entity x one view: the closure at visibility/mod.rs:788-858 */
static inline int entity_visible_in_view(uint32_t r, const float *gt, const float *bounds, uint8_t f,
                                         uint64_t entity_layers, uint64_t view_layers,
                                         const uint32_t *range_mask, int range_view_index,
                                         const v4 *hs, int view_no_cpu_culling) {
    if (!(f & F_INHERITED_VISIBLE)) return 0;
    if (!(view_layers & entity_layers) && !layers_ext_intersect(r, g_current_view)) return 0;
    if ((f & F_HAS_VIS_RANGE) && range_mask) {
        if (range_view_index < 0 || range_view_index > 31) return 0;
        if (!((range_mask[r] >> range_view_index) & 1u)) return 0;
    }
    if (!(f & F_NO_FRUSTUM_CULLING) && !view_no_cpu_culling) {
        const float *b = bounds + (size_t)r * 6;
        if (f & F_HAS_AABB) {
            aff a = aff_load(gt + (size_t)r * 12);
            v3 c = V3(b[0], b[1], b[2]), he = V3(b[3], b[4], b[5]);
            v3 sc = aff_transform_point(&a, c);
            float radius = v3_length(m3_mul_v3(&a.m, he));   /* radius_vec3a, global_transform.rs:252-254 */
            if (!frustum_intersects_sphere(hs, sc, radius, 0)) return 0;
            if (!frustum_intersects_obb(hs, c, he, &a, 1, 0)) return 0;
        } else if (f & F_HAS_SPHERE) {
            v3 sc = (f & F_SPHERE_FROM_GT)
                        ? V3(gt[(size_t)r * 12 + 9], gt[(size_t)r * 12 + 10], gt[(size_t)r * 12 + 11])
                        : V3(b[0], b[1], b[2]);
            if (!frustum_intersects_sphere(hs, sc, b[3], 0)) return 0;
        }
    }
    return 1;
}

/*
 * reset_view_visibility + check_visibility_cpu_culling +
 * mark_newly_hidden_entities_invisible (visibility/mod.rs:733-737, 748-876, 908-918).
 *
 * vv[r]            in/out ViewVisibility byte (bit0 current, bit1 previous)
 * vv_changed[r]    out: Changed<ViewVisibility> would fire
 * layer_mask       per-row RenderLayers first block, or NULL (=> default layer 0 => mask 1)
 * range_mask       VisibleEntityRanges bitmask per row, or NULL (resource absent)
 * class_mask[r]    bit per VisibilityClass the entity is in (0 => no list entry)
 * view_planes      [V][6][4]; view_layers [V]; view_flags [V]; view_range_index [V] (int8, -1 none)
 * visible_rows     [V][n] out, sorted ascending by entity_bits; visible_count[V] out
 *                  (0xFFFFFFFF for an inactive view: its VisibleEntities are left untouched,
 *                  visibility/mod.rs:780-782)
 */
/* mark_newly_hidden_entities_invisible (visibility/mod.rs:908-918).  The light-visibility systems
 * (check_point_light_mesh_visibility, bevy_light/src/lib.rs:517) run between check_visibility and this pass and OR
 * into the same bytes: orc_set_defer_mark_newly_hidden(1) makes orc_cull stop before it so a test can run them. */
static int g_defer_mark_newly_hidden = 0;
ORC_API void orc_set_defer_mark_newly_hidden(int on) { g_defer_mark_newly_hidden = on; }
ORC_API void orc_mark_newly_hidden(uint32_t n, const uint8_t *flags, uint8_t *vv, uint8_t *vv_changed) {
    for (uint32_t r = 0; r < n; ++r) {
        if (flags[r] & F_NO_CPU_CULLING) continue;
        if ((vv[r] & 3u) == 2u) { vv[r] = 0; vv_changed[r] = 1; }
    }
}
ORC_API int orc_cull(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags,
                     const uint64_t *layer_mask, const uint32_t *range_mask, const uint8_t *class_mask,
                     const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed,
                     uint32_t n_views, const float *view_planes, const uint64_t *view_layers,
                     const uint8_t *view_flags, const int8_t *view_range_index,
                     uint32_t *visible_rows, uint32_t *visible_count) {
    uint8_t *old = (uint8_t *)malloc(n ? n : 1);
    memcpy(old, vv, n);
    /* reset_view_visibility: v = (v & 1) << 1, bypassing change detection */
    for (uint32_t r = 0; r < n; ++r)
        if (!(flags[r] & F_NO_CPU_CULLING)) vv[r] = (uint8_t)((vv[r] & 1u) << 1);
    memset(vv_changed, 0, n);
    sort_item *items = (sort_item *)malloc((size_t)(n ? n : 1) * sizeof(sort_item));
    for (uint32_t v = 0; v < n_views; ++v) {
        if (!(view_flags[v] & VIEW_ACTIVE)) { visible_count[v] = 0xFFFFFFFFu; continue; }
        v4 hs[6]; memcpy(hs, view_planes + (size_t)v * 24, sizeof hs);
        uint32_t cnt = 0;
        g_current_view = v;
        for (uint32_t r = 0; r < n; ++r) {
            uint8_t f = flags[r];
            if (f & F_NO_CPU_CULLING) continue;                 /* Without<NoCpuCulling> */
            uint64_t el = layer_mask ? layer_mask[r] : 1ull;
            if (!entity_visible_in_view(r, gt, bounds, f, el, view_layers[v], range_mask,
                                        view_range_index ? view_range_index[v] : -1, hs,
                                        (view_flags[v] & VIEW_NO_CPU_CULLING) != 0))
                continue;
            /* set_visible (visibility/mod.rs:292-306) */
            if (!(vv[r] & 1u)) {
                if (!(vv[r] & 2u)) vv_changed[r] = 1;
                vv[r] |= 1u;
            }
            if (class_mask[r]) { items[cnt].key = entity_bits[r]; items[cnt].row = r; cnt++; }
        }
        qsort(items, cnt, sizeof(sort_item), cmp_sort_item);    /* sort_unstable by Entity::to_bits */
        for (uint32_t i = 0; i < cnt; ++i) visible_rows[(size_t)v * n + i] = items[i].row;
        visible_count[v] = cnt;
    }
    /* mark_newly_hidden_entities_invisible */
    if (!g_defer_mark_newly_hidden) orc_mark_newly_hidden(n, flags, vv, vv_changed);
    free(items); free(old);
    return 0;
}

/* ------------------------------------------------------------------------ */
/* stage 3: cluster                                                          */
/* ------------------------------------------------------------------------ */
typedef struct {
    /* ClusterConfig (crates/bevy_light/src/cluster/mod.rs:107-139) */
    uint32_t config_kind;        /* 0 None, 1 Single, 2 XYZ, 3 FixedZ */
    uint32_t cfg_dims[3];        /* XYZ dimensions */
    uint32_t cfg_total, cfg_z_slices;       /* FixedZ */
    float    first_slice_depth;  /* ClusterZConfig */
    uint32_t far_z_mode;         /* 0 MaxClusterableObjectRange, 1 Constant */
    float    far_z_constant;
    uint32_t dynamic_resizing;
    uint32_t screen_w, screen_h; /* camera.physical_viewport_size(); 0 => None */
    uint32_t view_cluster_bindings_max_indices;  /* GlobalClusterSettings */
    /* camera */
    float camera_gt[12];         /* GlobalTransform of the view */
    float clip_from_view[16];
    float frustum[24];           /* the view's Frustum (6 half spaces) */
    uint64_t view_layers;
    /* Clusters feedback (cluster/mod.rs:143-166): has_* = Option is Some */
    uint32_t has_last_farthest_z; float last_farthest_z;
    uint32_t has_last_index_count; uint32_t last_index_count;
} orc_cluster_view_in;

typedef struct {
    uint32_t cleared;            /* clusters.clear() path taken */
    uint32_t tile_size[2];
    uint32_t dims[3];
    float near, far;
    uint32_t is_orthographic;
    float cluster_factors[2];
    float view_from_world[16];
    float view_from_world_scale[3];
    float view_from_world_scale_max;
    uint32_t total_index_count;  /* -> last_frame_total_cluster_index_count */
    float farthest_z;            /* -> last_frame_farthest_z */
} orc_cluster_view_out;

/* ClusterConfig::dimensions_for_screen_size (cluster/mod.rs:311-347) */
/* VisibleEntities::entities is one Vec<Entity> PER VisibilityClass (TypeIdHashMap<Vec<Entity>>,
 * crates/bevy_camera/src/visibility/mod.rs:344-347): a visible entity is pushed once for every class id in its
 * VisibilityClass (:846-857, thread-local queues merged per class :861-868), and every class list is sorted by
 * Entity::to_bits() at the end (:870-874).  class_mask bit k = "the entity's VisibilityClass contains class k" (the shim's
 * registry of TypeIds, at most 8).  `visible` = the rows one view found visible AND classed (orc_cull's list, any order).
 * out_rows[k * n_visible + i], out_count[k] for k in 0..8. */
ORC_API void orc_visible_entities_by_class(uint32_t n_visible, const uint32_t *visible, const uint8_t *class_mask,
                                           const uint64_t *entity_bits, uint32_t *out_rows, uint32_t *out_count) {
    sort_item *items = (sort_item *)malloc((size_t)(n_visible ? n_visible : 1) * sizeof(sort_item));
    for (uint32_t k = 0; k < 8; ++k) {
        uint32_t cnt = 0;
        for (uint32_t i = 0; i < n_visible; ++i) {                  /* for class_id in visibility_class.iter(): push */
            uint32_t r = visible[i];
            if (class_mask[r] & (1u << k)) { items[cnt].key = entity_bits[r]; items[cnt].row = r; cnt++; }
        }
        qsort(items, cnt, sizeof(sort_item), cmp_sort_item);        /* entities.sort_unstable() per class */
        for (uint32_t i = 0; i < cnt; ++i) out_rows[(size_t)k * n_visible + i] = items[i].row;
        out_count[k] = cnt;
    }
    free(items);
}

ORC_API void orc_cluster_dimensions_for_screen_size(uint32_t kind, const uint32_t *cfg_dims, uint32_t total,
                                                    uint32_t z_slices, uint32_t w, uint32_t h, uint32_t *out3) {
    if (kind == 0) { out3[0] = out3[1] = out3[2] = 0; return; }
    if (kind == 1) { out3[0] = out3[1] = out3[2] = 1; return; }
    if (kind == 2) { out3[0] = cfg_dims[0]; out3[1] = cfg_dims[1]; out3[2] = cfg_dims[2]; return; }
    float aspect = (float)w / (float)h;       /* AspectRatio::try_from_pixels -> w as f32 / h as f32 */
    if (total < z_slices) z_slices = total;
    float per_layer = (float)total / (float)z_slices;
    float y = sqrtf(per_layer / aspect);
    uint32_t x = f32_as_u32(y * aspect);
    uint32_t yi = f32_as_u32(y);
    if (x == 0) { x = 1; yi = f32_as_u32(per_layer); }
    if (yi == 0) { x = f32_as_u32(per_layer); yi = 1; }
    out3[0] = x; out3[1] = yi; out3[2] = z_slices;
}
static inline uint32_t u32_max(uint32_t a, uint32_t b) { return a > b ? a : b; }
static inline uint32_t u32_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
/* Clusters::update (cluster/mod.rs:398-416) */
ORC_API void orc_clusters_update(uint32_t w, uint32_t h, const uint32_t *req3, uint32_t *tile2, uint32_t *dims3) {
    tile2[0] = u32_max(f32_as_u32(ceilf((float)w / (float)req3[0])), 1u);
    tile2[1] = u32_max(f32_as_u32(ceilf((float)h / (float)req3[1])), 1u);
    dims3[0] = u32_max(f32_as_u32(ceilf((float)w / (float)tile2[0])), 1u);
    dims3[1] = u32_max(f32_as_u32(ceilf((float)h / (float)tile2[1])), 1u);
    dims3[2] = u32_max(req3[2], 1u);
}
/* calculate_cluster_factors (assign.rs:817-832) */
static inline void cluster_factors(float near, float far, float z_slices, int ortho, float *out2) {
    if (ortho) { out2[0] = -near; out2[1] = z_slices / (-far - -near); }
    else {
        float k = (z_slices - 1.0f) / logf(far / near);
        out2[0] = k; out2[1] = logf(near) * k;
    }
}
/* z_slice_to_view_z (assign.rs:903-920) */
static inline float z_slice_to_view_z(float near, float far, uint32_t z_slices, uint32_t z_slice, int ortho) {
    if (ortho) return -near - (far - near) * (float)z_slice / (float)z_slices;
    if (z_slice == 0) return 0.0f;
    return -near * powf(far / near, (float)(z_slice - 1) / (float)(z_slices - 1));
}
/* view_z_to_z_slice (assign.rs:1046-1062) */
static inline uint32_t view_z_to_z_slice(const float *f, uint32_t z_slices, float view_z, int ortho) {
    uint32_t z = ortho ? f32_as_u32(floorf((view_z - f[0]) * f[1]))
                       : f32_as_u32(logf(-view_z) * f[0] - f[1] + 1.0f);
    return u32_min(z, z_slices - 1);
}
/* ndc_position_to_cluster (assign.rs:922-941) */
static inline void ndc_position_to_cluster(const uint32_t *dims, const float *factors, int ortho,
                                           v3 ndc, float view_z, uint32_t *out) {
    float fx = gl_min(gl_max(ndc.x * 0.5f + 0.5f, 0.0f), 1.0f);
    float fy = gl_min(gl_max(ndc.y * -0.5f + 0.5f, 0.0f), 1.0f);
    float x = floorf(fx * (float)dims[0]), y = floorf(fy * (float)dims[1]);
    uint32_t z = view_z_to_z_slice(factors, dims[2], view_z, ortho);
    out[0] = u32_min(f32_as_u32(x), dims[0] - 1);
    out[1] = u32_min(f32_as_u32(y), dims[1] - 1);
    out[2] = u32_min(z, dims[2] - 1);
}
/* clip_to_view (assign.rs:1064-1067) */
static inline v4 clip_to_view(const m4 *view_from_clip, v4 clip) {
    v4 view = m4_mul_v4(view_from_clip, clip);
    return V4(view.x / view.w, view.y / view.w, view.z / view.w, view.w / view.w);
}
static inline v3 v3_div_s(v3 a, float s) { return V3(a.x / s, a.y / s, a.z / s); }

/* cluster_space_clusterable_object_aabb (assign.rs:948-1036) */
static void cluster_space_aabb(const m4 *vfw, v3 vfw_scale, const m4 *cfv, v3 center, float radius,
                               v3 *out_min, v3 *out_max) {
    v3 c = v4_xyz(m4_mul_v4(vfw, v3_extend(center, 1.0f)));
    v3 he = v3_scale(v3_abs(vfw_scale), radius);       /* radius * scale.abs() (f32 * Vec3) */
    v3 vmin = v3_sub(c, he), vmax = v3_add(c, he);
    vmin.z = fminf(vmin.z, -1.17549435e-38f);          /* f32::min with -f32::MIN_POSITIVE */
    vmax.z = fminf(vmax.z, -1.17549435e-38f);
    v3 a = vmin, b = V3(vmin.x, vmin.y, vmax.z), c2 = V3(vmax.x, vmax.y, vmin.z), d = vmax;
    v4 ca = m4_mul_v4(cfv, v3_extend(a, 1.0f)), cb = m4_mul_v4(cfv, v3_extend(b, 1.0f));
    v4 cc = m4_mul_v4(cfv, v3_extend(c2, 1.0f)), cd = m4_mul_v4(cfv, v3_extend(d, 1.0f));
    v3 na = v3_div_s(v4_xyz(ca), ca.w), nb = v3_div_s(v4_xyz(cb), cb.w);
    v3 nc = v3_div_s(v4_xyz(cc), cc.w), nd = v3_div_s(v4_xyz(cd), cd.w);
    v3 nmin = v3_min(v3_min(v3_min(na, nb), nc), nd);
    v3 nmax = v3_max(v3_max(v3_max(na, nb), nc), nd);
    /* Vec2::clamp(NDC_MIN, NDC_MAX) = max(min).min(max) */
    out_min->x = gl_min(gl_max(nmin.x, -1.0f), 1.0f); out_min->y = gl_min(gl_max(nmin.y, -1.0f), 1.0f);
    out_max->x = gl_min(gl_max(nmax.x, -1.0f), 1.0f); out_max->y = gl_min(gl_max(nmax.y, -1.0f), 1.0f);
    out_min->z = vmin.z; out_max->z = vmax.z;
}

typedef struct { v3 c; float r; } sph;
/* project_to_plane_z (assign.rs:1094-1113) */
static inline int project_to_plane_z(sph *o, v4 plane) {
    float z = plane.w / plane.z;
    float d = z - o->c.z;
    if (fabsf(d) > o->r) return 0;
    o->c.z = z;
    o->r = sqrtf(o->r * o->r - d * d);
    return 1;
}
/* project_to_plane_y (assign.rs:1116-1134) */
static inline int project_to_plane_y(sph *o, v4 plane, int ortho) {
    /* Vec2 dot (scalar): x*x' + y*y' over (y,z) */
    float d = ortho ? plane.w - o->c.y : -(o->c.y * plane.y + o->c.z * plane.z);
    if (fabsf(d) > o->r) return 0;
    o->c = v3_add(o->c, V3(d * plane.x, d * plane.y, d * plane.z));   /* f32 * Vec3A */
    o->r = sqrtf(o->r * o->r - d * d);
    return 1;
}
/* get_distance_x (assign.rs:1081-1091) */
static inline float get_distance_x(v4 plane, v3 p, int ortho) {
    return ortho ? p.x - plane.w : plane.x * p.x + plane.z * p.z;
}

/*
 * assign_objects_to_clusters for ONE view, point lights only
 * (crates/bevy_light/src/cluster/assign.rs:324-811).
 *
 * lights: n_lights x { pos[3], range } already filtered to view_visibility.get()
 *         (assign.rs:193-210) in query order; light_layers[n_lights] (or NULL => 1).
 * Output: per-cluster lists in CSR form.  offsets[n_clusters+1]; indices =
 *         light ordinals (position in `lights`), in push order (light-major).
 *         indices_cap bounds the indices buffer.
 * plane outputs (may be NULL): x_planes[(dims.x+1)*4], y_planes, z_planes.
 */
ORC_API int orc_assign_lights_to_clusters(const orc_cluster_view_in *in, uint32_t n_lights,
                                          const float *lights, const uint64_t *light_layers,
                                          orc_cluster_view_out *out, uint32_t *offsets /* 4097 */,
                                          uint32_t *indices, uint32_t indices_cap,
                                          float *x_planes_out, float *y_planes_out, float *z_planes_out) {
    memset(out, 0, sizeof *out);
    /* ClusterConfig::None or zero-sized viewport => clusters.clear() (assign.rs:329-340) */
    if (in->config_kind == 0 || in->screen_w == 0 || in->screen_h == 0) {
        out->cleared = 1; out->tile_size[0] = out->tile_size[1] = 1;
        offsets[0] = 0;
        return 0;
    }
    uint32_t req[3];
    orc_cluster_dimensions_for_screen_size(in->config_kind, in->cfg_dims, in->cfg_total, in->cfg_z_slices,
                                           in->screen_w, in->screen_h, req);
    aff cam = aff_load(in->camera_gt);
    m4 cfv = m4_load(in->clip_from_view);
    /* compute_transform().scale.recip()  (GlobalTransform::scale via to_scale_rotation_translation:
     * glam Affine3A::to_scale_rotation_translation: det = matrix3.determinant();
     * scale = (x.length()*signum(det), y.length(), z.length())) */
    float det = v3_dot(cam.m.z, v3_cross(cam.m.x, cam.m.y));
    float sgn = copysignf(1.0f, det);  /* math::signum; NaN not modelled */
    v3 scale = V3(v3_length(cam.m.x) * sgn, v3_length(cam.m.y), v3_length(cam.m.z));
    v3 vfw_scale = V3(1.0f / scale.x, 1.0f / scale.y, 1.0f / scale.z);
    float vfw_scale_max = gl_max(gl_max(fabsf(vfw_scale.x), fabsf(vfw_scale.y)), fabsf(vfw_scale.z));
    aff inv = aff_inverse(&cam);
    m4 vfw = m4_from_aff(&inv);
    int ortho = cfv.w.w == 1.0f;
    float cfg_first = (in->config_kind == 1) ? 0.0f : in->first_slice_depth;
    uint32_t far_mode = (in->config_kind == 1) ? 0u : in->far_z_mode;
    float far_z = far_mode == 0 ? (in->has_last_farthest_z ? in->last_farthest_z : 1000.0f) : in->far_z_constant;
    float first_slice_depth;
    if (ortho) first_slice_depth = (cfv.w.z - 1.0f) / cfv.z.z;
    else if (req[2] == 1) first_slice_depth = fmaxf(cfg_first, far_z);
    else first_slice_depth = cfg_first;
    first_slice_depth = first_slice_depth * vfw_scale.z;
    far_z = fmaxf(far_z, first_slice_depth);
    float factors[2];
    cluster_factors(first_slice_depth, far_z, (float)req[2], ortho, factors);
    int dyn = (in->config_kind >= 2) && in->dynamic_resizing;
    if (dyn && in->has_last_index_count && in->last_index_count > in->view_cluster_bindings_max_indices) {
        float index_ratio = (float)in->view_cluster_bindings_max_indices / (float)in->last_index_count;
        float xy_ratio = sqrtf(index_ratio);
        req[0] = u32_max(f32_as_u32(floorf((float)req[0] * xy_ratio)), 1u);
        req[1] = u32_max(f32_as_u32(floorf((float)req[1] * xy_ratio)), 1u);
    }
    uint32_t dims[3], tile[2];
    orc_clusters_update(in->screen_w, in->screen_h, req, tile, dims);
    out->tile_size[0] = tile[0]; out->tile_size[1] = tile[1];
    out->dims[0] = dims[0]; out->dims[1] = dims[1]; out->dims[2] = dims[2];
    out->near = first_slice_depth; out->far = far_z;
    out->is_orthographic = (uint32_t)ortho;
    out->cluster_factors[0] = factors[0]; out->cluster_factors[1] = factors[1];
    m4_store(out->view_from_world, &vfw);
    out->view_from_world_scale[0] = vfw_scale.x; out->view_from_world_scale[1] = vfw_scale.y;
    out->view_from_world_scale[2] = vfw_scale.z; out->view_from_world_scale_max = vfw_scale_max;
    uint32_t n_clusters = dims[0] * dims[1] * dims[2];
    if (n_clusters > 4096) return -3;   /* debug_assert in the reference (assign.rs:410-413) */
    m4 vfc = m4_inverse(&cfv);

    v4 *xp = (v4 *)malloc(sizeof(v4) * (dims[0] + 1));
    v4 *yp = (v4 *)malloc(sizeof(v4) * (dims[1] + 1));
    v4 *zp = (v4 *)malloc(sizeof(v4) * (dims[2] + 1));
    /* plane tables (assign.rs:429-485) */
    for (uint32_t x = 0; x <= dims[0]; ++x) {
        float prop = (float)x / (float)dims[0];
        float x_pos = prop * 2.0f - 1.0f;
        if (ortho) {
            float view_x = clip_to_view(&vfc, V4(x_pos, 0.0f, 1.0f, 1.0f)).x;
            xp[x] = half_space_new(V4(1.0f, 0.0f, 0.0f, view_x * 1.0f));
        } else {
            v3 nb = v4_xyz(clip_to_view(&vfc, V4(x_pos, -1.0f, 1.0f, 1.0f)));
            v3 nt = v4_xyz(clip_to_view(&vfc, V4(x_pos, 1.0f, 1.0f, 1.0f)));
            v3 normal = v3_cross(nb, nt);
            xp[x] = half_space_new(v3_extend(normal, v3_dot(nb, normal)));
        }
    }
    for (uint32_t y = 0; y <= dims[1]; ++y) {
        float prop = 1.0f - (float)y / (float)dims[1];
        float y_pos = prop * 2.0f - 1.0f;
        if (ortho) {
            float view_y = clip_to_view(&vfc, V4(0.0f, y_pos, 1.0f, 1.0f)).y;
            yp[y] = half_space_new(V4(0.0f, 1.0f, 0.0f, view_y * 1.0f));
        } else {
            v3 nl = v4_xyz(clip_to_view(&vfc, V4(-1.0f, y_pos, 1.0f, 1.0f)));
            v3 nr = v4_xyz(clip_to_view(&vfc, V4(1.0f, y_pos, 1.0f, 1.0f)));
            v3 normal = v3_cross(nr, nl);
            yp[y] = half_space_new(v3_extend(normal, v3_dot(nr, normal)));
        }
    }
    for (uint32_t z = 0; z <= dims[2]; ++z) {
        float view_z = z_slice_to_view_z(first_slice_depth, far_z, dims[2], z, ortho);
        /* normal = -Vec3::Z ; d = view_z * normal.z */
        zp[z] = half_space_new(V4(-0.0f, -0.0f, -1.0f, view_z * -1.0f));
    }
    if (x_planes_out) memcpy(x_planes_out, xp, sizeof(v4) * (dims[0] + 1));
    if (y_planes_out) memcpy(y_planes_out, yp, sizeof(v4) * (dims[1] + 1));
    if (z_planes_out) memcpy(z_planes_out, zp, sizeof(v4) * (dims[2] + 1));

    /* per-cluster growable lists: first count, then fill (two passes over the same
     * deterministic loop) */
    uint32_t *counts = (uint32_t *)calloc(n_clusters + 1, sizeof(uint32_t));
    uint32_t total = 0; float farthest_z = 0.0f;
    v4 row2 = m4_row(&vfw, 2);
    v4 frustum[6]; memcpy(frustum, in->frustum, sizeof frustum);
    int rc = 0;
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1) {
            offsets[0] = 0;
            for (uint32_t c = 0; c < n_clusters; ++c) offsets[c + 1] = offsets[c] + counts[c];
            if (offsets[n_clusters] > indices_cap) { rc = -4; break; }
            memset(counts, 0, sizeof(uint32_t) * n_clusters);
        }
        for (uint32_t li = 0; li < n_lights; ++li) {
            uint64_t ll = light_layers ? light_layers[li] : 1ull;
            if (!(in->view_layers & ll)) continue;                                  /* assign.rs:489 */
            v3 lc = V3(lights[li * 4 + 0], lights[li * 4 + 1], lights[li * 4 + 2]);
            float range = lights[li * 4 + 3];
            if (!frustum_intersects_sphere(frustum, lc, range, 1)) continue;        /* assign.rs:496 */
            v3 amin, amax;
            cluster_space_aabb(&vfw, vfw_scale, &cfv, lc, range, &amin, &amax);
            uint32_t cmin[3], cmax[3];
            ndc_position_to_cluster(dims, factors, ortho, amin, amin.z, cmin);
            ndc_position_to_cluster(dims, factors, ortho, amax, amax.z, cmax);
            uint32_t lo[3], hi[3];
            for (int k = 0; k < 3; ++k) { lo[k] = u32_min(cmin[k], cmax[k]); hi[k] = u32_max(cmin[k], cmax[k]); }
            sph vs;
            vs.c = v4_xyz(m4_mul_v4(&vfw, v3_extend(lc, 1.0f)));
            vs.r = range * vfw_scale_max;
            if (pass == 0) {
                float this_far = -v4_dot(row2, v3_extend(lc, 1.0f)) + range * vfw_scale.z;
                farthest_z = fmaxf(farthest_z, this_far);
            }
            v4 cclip = m4_mul_v4(&cfv, v3_extend(vs.c, 1.0f));
            v3 cndc = v3_div_s(v4_xyz(cclip), cclip.w);
            uint32_t cc[3];
            ndc_position_to_cluster(dims, factors, ortho, cndc, vs.c.z, cc);
            int has_zc = cndc.z <= 1.0f; uint32_t zc = cc[2];
            int has_yc; uint32_t yc = 0;
            if (cndc.y > 1.0f) has_yc = 0;
            else if (cndc.y < -1.0f) { has_yc = 1; yc = dims[1] + 1; }
            else { has_yc = 1; yc = cc[1]; }
            for (uint32_t z = lo[2]; z <= hi[2]; ++z) {
                sph zo = vs;
                if (!has_zc || z != zc) {
                    v4 zpl = (has_zc && z < zc) ? zp[z + 1] : zp[z];
                    if (!project_to_plane_z(&zo, zpl)) continue;
                }
                for (uint32_t y = lo[1]; y <= hi[1]; ++y) {
                    sph yo = zo;
                    if (!has_yc || y != yc) {
                        v4 ypl = (has_yc && y < yc) ? yp[y + 1] : yp[y];
                        if (!project_to_plane_y(&yo, ypl, ortho)) continue;
                    }
                    uint32_t min_x = lo[0];
                    while (1) {
                        if (min_x >= hi[0] || -get_distance_x(xp[min_x + 1], yo.c, ortho) + yo.r > 0.0f) break;
                        min_x++;
                    }
                    uint32_t max_x = hi[0];
                    while (1) {
                        if (max_x <= min_x || get_distance_x(xp[max_x], yo.c, ortho) + yo.r > 0.0f) break;
                        max_x--;
                    }
                    uint32_t ci = (y * dims[0] + min_x) * dims[2] + z;
                    for (uint32_t x = min_x; x <= max_x; ++x) {
                        if (pass == 1) indices[offsets[ci] + counts[ci]] = li;
                        counts[ci]++;
                        ci += dims[2];
                    }
                    if (pass == 0) total += max_x - min_x + 1;
                }
            }
        }
    }
    out->total_index_count = total;
    out->farthest_z = farthest_z;
    free(counts); free(xp); free(yp); free(zp);
    return rc;
}

/* libm entry points re-exported so tests can pin the host-side thresholds */
ORC_API float orc_logf(float x) { return logf(x); }
ORC_API float orc_powf(float x, float y) { return powf(x, y); }
ORC_API uint32_t orc_view_z_to_z_slice(const float *factors2, uint32_t z_slices, float view_z, int ortho) {
    return view_z_to_z_slice(factors2, z_slices, view_z, ortho);
}


/* ------------------------------------------------------------------------ */
/* SURVEY.md 8(f) N3: shadow-view culling for point lights                   */
/* ------------------------------------------------------------------------ */
/* Quat::from_rotation_axes (glam f32/scalar quat.rs; Quat::from_mat3 forwards the three columns).
 * PARITY UNPINNED: restated from glam's published algorithm, no reference vector exercises it. */
static v4 quat_from_rotation_axes(v3 xa, v3 ya, v3 za) {
    float m00 = xa.x, m01 = xa.y, m02 = xa.z, m10 = ya.x, m11 = ya.y, m12 = ya.z, m20 = za.x, m21 = za.y, m22 = za.z;
    if (m22 <= 0.0f) {                       /* x^2 + y^2 >= z^2 + w^2 */
        float dif10 = m11 - m00, omm22 = 1.0f - m22;
        if (dif10 <= 0.0f) {                 /* x^2 >= y^2 */
            float four_xsq = omm22 - dif10, inv4x = 0.5f / sqrtf(four_xsq);
            return V4(four_xsq * inv4x, (m01 + m10) * inv4x, (m02 + m20) * inv4x, (m12 - m21) * inv4x);
        } else {                             /* y^2 >= x^2 */
            float four_ysq = omm22 + dif10, inv4y = 0.5f / sqrtf(four_ysq);
            return V4((m01 + m10) * inv4y, four_ysq * inv4y, (m12 + m21) * inv4y, (m20 - m02) * inv4y);
        }
    } else {                                 /* z^2 + w^2 >= x^2 + y^2 */
        float sum10 = m11 + m00, opm22 = 1.0f + m22;
        if (sum10 <= 0.0f) {                 /* z^2 >= w^2 */
            float four_zsq = opm22 - sum10, inv4z = 0.5f / sqrtf(four_zsq);
            return V4((m02 + m20) * inv4z, (m12 + m21) * inv4z, four_zsq * inv4z, (m01 - m10) * inv4z);
        } else {                             /* w^2 >= z^2 */
            float four_wsq = opm22 + sum10, inv4w = 0.5f / sqrtf(four_wsq);
            return V4((m12 - m21) * inv4w, (m20 - m02) * inv4w, (m01 - m10) * inv4w, four_wsq * inv4w);
        }
    }
}
/* Transform::IDENTITY.looking_at(target, up) -> look_to (transform.rs:475-484); Dir3::new = v / |v|,
 * try_normalize = v * (1 / |v|) -- both exact for the axis-aligned CUBE_MAP_FACES */
static v4 look_to_rotation(v3 direction, v3 up_in) {
    float dl = v3_length(direction), ul = v3_length(up_in);
    v3 back = v3_neg(v3_div_s(direction, dl));
    v3 up = v3_div_s(up_in, ul);
    v3 right = v3_cross(up, back);
    right = v3_scale(right, 1.0f / v3_length(right));
    up = v3_cross(back, right);
    return quat_from_rotation_axes(right, up, back);
}
/* update_point_light_frusta (crates/bevy_light/src/point_light.rs:212-265) for one light: planes[6][6][4] */
ORC_API void orc_point_light_frusta(const float *light_gt12, float range, float shadow_map_near_z, float *planes) {
    static const float faces[6][6] = {   /* CUBE_MAP_FACES target, up (bevy_camera/src/primitives.rs:348-379) */
        {1, 0, 0, 0, 1, 0}, {-1, 0, 0, 0, 1, 0}, {0, 1, 0, 0, 0, 1}, {0, -1, 0, 0, 0, -1}, {0, 0, -1, 0, 1, 0}, {0, 0, 1, 0, 1, 0}};
    aff light = aff_load(light_gt12);
    float cfv16[16];
    orc_perspective_infinite_reverse_rh(1.57079632679489661923f, 1.0f, shadow_map_near_z, cfv16);   /* FRAC_PI_2 */
    m4 cfv = m4_load(cfv16);
    v3 view_backward = gt_back(&light);
    for (int f = 0; f < 6; ++f) {
        v4 q = look_to_rotation(V3(faces[f][0], faces[f][1], faces[f][2]), V3(faces[f][3], faces[f][4], faces[f][5]));
        /* world_from_view = Transform::from_translation(t) * view_rotation: rotation IDENTITY * q = q, scale 1, translation t */
        float trs[10] = {light.t.x, light.t.y, light.t.z, q.x, q.y, q.z, q.w, 1.0f, 1.0f, 1.0f};
        aff wfv = aff_from_trs(trs), inv = aff_inverse(&wfv);
        m4 vfw = m4_from_aff(&inv);
        m4 cfw = m4_mul(&cfv, &vfw);
        v4 hs[6];
        view_frustum_custom_far(&cfw, light.t, view_backward, range, hs);
        memcpy(planes + (size_t)f * 24, hs, sizeof hs);
    }
}
/* check_point_light_mesh_visibility, point-light half (crates/bevy_light/src/lib.rs:517-668).
 * caster[r] != 0: the row is in visible_entity_query (Mesh3d, no NotShadowCaster, no DirectionalLight);
 * NoCpuCulling comes from flags.  The caller passes the lights that are in some view's VisibleEntities and have
 * shadow_maps_enabled (:561-580): light_sphere[L][4] = GlobalTransform translation, range; frusta[L][6][6][4].
 * lod_origin_index: bit of get_shadow_lod_origin's view in the range masks, -1 = none / not in the views map.
 * vv / vv_changed: in the state check_visibility left them (before mark_newly_hidden).
 * Out: visible_rows[(l*6+face)*n ...] ascending by entity bits (sort_unstable, :650-661), visible_count[L*6]. */
ORC_API int orc_check_point_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags,
                                                  const uint8_t *caster, const uint64_t *layer_mask, const uint32_t *range_mask,
                                                  int lod_origin_index, const uint64_t *entity_bits, uint8_t *vv,
                                                  uint8_t *vv_changed, uint32_t n_lights, const float *light_sphere,
                                                  const uint64_t *light_layers, const float *frusta, uint32_t *visible_rows,
                                                  uint32_t *visible_count) {
    sort_item *items = (sort_item *)malloc((size_t)(n ? n : 1) * 6 * sizeof(sort_item));
    if (!items) return 1;
    for (uint32_t l = 0; l < n_lights; ++l) {
        uint32_t cnt[6] = {0, 0, 0, 0, 0, 0};
        const uint64_t view_mask = light_layers ? light_layers[l] : 1ull;
        const float *ls = light_sphere + (size_t)l * 4;
        v4 hs[6][6]; memcpy(hs, frusta + (size_t)l * 144, sizeof hs);
        for (uint32_t r = 0; r < n; ++r) {
            const uint8_t f = flags[r];
            if (!caster[r] || (f & F_NO_CPU_CULLING)) continue;
            if (!(f & F_INHERITED_VISIBLE)) continue;
            if (!(view_mask & (layer_mask ? layer_mask[r] : 1ull))) continue;
            if ((f & F_HAS_VIS_RANGE) && range_mask &&
                (lod_origin_index < 0 || lod_origin_index > 31 || !((range_mask[r] >> lod_origin_index) & 1u)))
                continue;
            int face_vis[6] = {1, 1, 1, 1, 1, 1};
            if (f & F_HAS_AABB) {   /* (Some(aabb), Some(transform)) */
                const float *b = bounds + (size_t)r * 6;
                const int no_fc = (f & F_NO_FRUSTUM_CULLING) != 0;
                if (!no_fc && !orc_sphere_intersects_obb(ls, ls[3], b, b + 3, gt + (size_t)r * 12)) continue;
                aff a = aff_load(gt + (size_t)r * 12);
                for (int k = 0; k < 6; ++k)
                    face_vis[k] = no_fc || frustum_intersects_obb(hs[k], V3(b[0], b[1], b[2]), V3(b[3], b[4], b[5]), &a, 1, 1);
            }
            for (int k = 0; k < 6; ++k) {
                if (!face_vis[k]) continue;
                if (!(vv[r] & 1u)) {   /* set_visible (visibility/mod.rs:292-306) */
                    if (!(vv[r] & 2u)) vv_changed[r] = 1;
                    vv[r] |= 1u;
                }
                items[(size_t)k * n + cnt[k]].key = entity_bits[r]; items[(size_t)k * n + cnt[k]].row = r; cnt[k]++;
            }
        }
        for (int k = 0; k < 6; ++k) {
            qsort(items + (size_t)k * n, cnt[k], sizeof(sort_item), cmp_sort_item);
            uint32_t *dst = visible_rows + ((size_t)l * 6 + k) * n;
            for (uint32_t i = 0; i < cnt[k]; ++i) dst[i] = items[(size_t)k * n + i].row;
            visible_count[l * 6 + k] = cnt[k];
        }
    }
    free(items);
    return 0;
}

/* check_point_light_mesh_visibility, spot-light half (crates/bevy_light/src/lib.rs:670-748): one Frustum per light
 * (near and far planes checked), the same range-sphere pre-test and gates as the point-light half.
 * Out: visible_rows[l*n ...] ascending by entity bits, visible_count[L].  (Device side: not built yet.) */
ORC_API int orc_check_spot_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags,
                                                 const uint8_t *caster, const uint64_t *layer_mask, const uint32_t *range_mask,
                                                 int lod_origin_index, const uint64_t *entity_bits, uint8_t *vv,
                                                 uint8_t *vv_changed, uint32_t n_lights, const float *light_sphere,
                                                 const uint64_t *light_layers, const float *frusta, uint32_t *visible_rows,
                                                 uint32_t *visible_count) {
    sort_item *items = (sort_item *)malloc((size_t)(n ? n : 1) * sizeof(sort_item));
    if (!items) return 1;
    for (uint32_t l = 0; l < n_lights; ++l) {
        uint32_t cnt = 0;
        const uint64_t view_mask = light_layers ? light_layers[l] : 1ull;
        const float *ls = light_sphere + (size_t)l * 4;
        v4 hs[6]; memcpy(hs, frusta + (size_t)l * 24, sizeof hs);
        for (uint32_t r = 0; r < n; ++r) {
            const uint8_t f = flags[r];
            if (!caster[r] || (f & F_NO_CPU_CULLING) || !(f & F_INHERITED_VISIBLE)) continue;
            if (!(view_mask & (layer_mask ? layer_mask[r] : 1ull))) continue;
            if ((f & F_HAS_VIS_RANGE) && range_mask &&
                (lod_origin_index < 0 || lod_origin_index > 31 || !((range_mask[r] >> lod_origin_index) & 1u)))
                continue;
            if (f & F_HAS_AABB) {
                const float *b = bounds + (size_t)r * 6;
                const int no_fc = (f & F_NO_FRUSTUM_CULLING) != 0;
                if (!no_fc && !orc_sphere_intersects_obb(ls, ls[3], b, b + 3, gt + (size_t)r * 12)) continue;
                aff a = aff_load(gt + (size_t)r * 12);
                if (!(no_fc || frustum_intersects_obb(hs, V3(b[0], b[1], b[2]), V3(b[3], b[4], b[5]), &a, 1, 1))) continue;
            }
            if (!(vv[r] & 1u)) { if (!(vv[r] & 2u)) vv_changed[r] = 1; vv[r] |= 1u; }   /* set_visible */
            items[cnt].key = entity_bits[r]; items[cnt].row = r; cnt++;
        }
        qsort(items, cnt, sizeof(sort_item), cmp_sort_item);
        for (uint32_t i = 0; i < cnt; ++i) visible_rows[(size_t)l * n + i] = items[i].row;
        visible_count[l] = cnt;
    }
    free(items);
    return 0;
}
/* check_dir_light_mesh_visibility (crates/bevy_light/src/lib.rs:342-510) for the (directional light, view) pairs whose
 * light has shadow_maps_enabled and is visible (:395-399): item i has n_cascades[i] frusta (CascadesFrusta of that
 * view, concatenated in `frusta`), the light's RenderLayers and the view's bit in the VisibleEntityRanges masks
 * (-1 = the view is not in the map => entity_is_in_range_of_view is false).  The near plane is NOT tested (a caster may
 * lie before it, :455-458).  Out: per cascade (in item order) rows ascending by entity bits; set_visible is applied
 * (the reference defers it to a command, same result).  Device side: cascade items of b200vis_set_shadow_items (k_shadow_cull). */
ORC_API int orc_check_dir_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags,
                                                const uint8_t *caster, const uint64_t *layer_mask, const uint32_t *range_mask,
                                                const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed, uint32_t n_items,
                                                const int32_t *view_range_index, const uint64_t *light_layers,
                                                const uint32_t *n_cascades, const float *frusta, uint32_t *visible_rows,
                                                uint32_t *visible_count) {
    sort_item *items = (sort_item *)malloc((size_t)(n ? n : 1) * sizeof(sort_item));
    uint8_t *hit = (uint8_t *)malloc(n ? n : 1);
    if (!items || !hit) { free(items); free(hit); return 1; }
    uint32_t casc0 = 0;
    for (uint32_t it = 0; it < n_items; ++it) {
        const uint64_t view_mask = light_layers ? light_layers[it] : 1ull;
        const int vri = view_range_index ? view_range_index[it] : -1;
        for (uint32_t c = 0; c < n_cascades[it]; ++c) {
            v4 hs[6]; memcpy(hs, frusta + (size_t)(casc0 + c) * 24, sizeof hs);
            uint32_t cnt = 0;
            for (uint32_t r = 0; r < n; ++r) {
                const uint8_t f = flags[r];
                hit[r] = 0;
                if (!caster[r] || (f & F_NO_CPU_CULLING) || !(f & F_INHERITED_VISIBLE)) continue;
                if (!(view_mask & (layer_mask ? layer_mask[r] : 1ull))) continue;
                if ((f & F_HAS_VIS_RANGE) && range_mask && (vri < 0 || vri > 31 || !((range_mask[r] >> vri) & 1u))) continue;
                if (f & F_HAS_AABB) {
                    const float *b = bounds + (size_t)r * 6;
                    aff a = aff_load(gt + (size_t)r * 12);
                    if (!(f & F_NO_FRUSTUM_CULLING) &&
                        !frustum_intersects_obb(hs, V3(b[0], b[1], b[2]), V3(b[3], b[4], b[5]), &a, 0, 1))
                        continue;
                }
                hit[r] = 1;
                items[cnt].key = entity_bits[r]; items[cnt].row = r; cnt++;
            }
            for (uint32_t r = 0; r < n; ++r)
                if (hit[r] && !(vv[r] & 1u)) { if (!(vv[r] & 2u)) vv_changed[r] = 1; vv[r] |= 1u; }
            qsort(items, cnt, sizeof(sort_item), cmp_sort_item);
            for (uint32_t i = 0; i < cnt; ++i) visible_rows[(size_t)(casc0 + c) * n + i] = items[i].row;
            visible_count[casc0 + c] = cnt;
        }
        casc0 += n_cascades[it];
    }
    free(items); free(hit);
    return 0;
}
