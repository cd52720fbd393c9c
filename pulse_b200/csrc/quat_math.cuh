// Device-side xyzw quaternion algebra for the HumanoidIm step path.
//
// Each routine restates the arithmetic of a reference function (cited) in per-lane scalar form.
// Where the reference's result feeds an INTEGER output (frame indices, reset masks) the exact fp32
// operation order is reproduced with round-to-nearest intrinsics so FMA contraction cannot change
// the result; everything else is free to contract (tolerance 1e-4 on observations / rewards).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace pulse {

struct Vec3 {
  float x, y, z;
};
struct Quat {
  float x, y, z, w;
};

__device__ __forceinline__ Vec3 operator-(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ Vec3 operator+(Vec3 a, Vec3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ float dot3(Vec3 a, Vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float sq3(Vec3 a) { return a.x * a.x + a.y * a.y + a.z * a.z; }

__device__ __forceinline__ Vec3 ldv(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ Quat ldq(const float* p) { return {p[0], p[1], p[2], p[3]}; }
// one 16-byte load: p must be 16-byte aligned
__device__ __forceinline__ Quat ldq4(const float* p) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  return {v.x, v.y, v.z, v.w};
}
__device__ __forceinline__ void stv(float* o, Vec3 v) {
  o[0] = v.x;
  o[1] = v.y;
  o[2] = v.z;
}

// isaacgym.torch_utils.quat_mul [3P-memory]: 8-multiplication Hamilton product.
__device__ __forceinline__ Quat qmul(Quat a, Quat b) {
  float ww = (a.z + a.x) * (b.x + b.y);
  float yy = (a.w - a.y) * (b.w + b.z);
  float zz = (a.w + a.y) * (b.w - b.z);
  float xx = ww + yy + zz;
  float qq = 0.5f * (xx + (a.z - a.x) * (b.x - b.y));
  Quat r;
  r.w = qq - ww + (a.z - a.y) * (b.y - b.z);
  r.x = qq - xx + (a.x + a.w) * (b.x + b.w);
  r.y = qq - yy + (a.w - a.x) * (b.y + b.z);
  r.z = qq - zz + (a.z + a.y) * (b.w - b.x);
  return r;
}

__device__ __forceinline__ Quat qconj(Quat a) { return {-a.x, -a.y, -a.z, a.w}; }

// humanoid.py:1617-1620 (remove_base_rot): q (x) conj(0.5, 0.5, 0.5, 0.5), skipped for an upright start
__device__ __forceinline__ Quat base_rot_removed(Quat q, bool upright) {
  return upright ? q : qmul(q, Quat{-0.5f, -0.5f, -0.5f, 0.5f});
}

// phc/utils/torch_utils.py:45-55 (my_quat_rotate)
__device__ __forceinline__ Vec3 qrot(Quat q, Vec3 v) {
  float s = 2.0f * q.w * q.w - 1.0f;
  float d = 2.0f * (q.x * v.x + q.y * v.y + q.z * v.z);
  float w2 = 2.0f * q.w;
  Vec3 c = {q.y * v.z - q.z * v.y, q.z * v.x - q.x * v.z, q.x * v.y - q.y * v.x};
  return {v.x * s + c.x * w2 + q.x * d, v.y * s + c.y * w2 + q.y * d, v.z * s + c.z * w2 + q.z * d};
}

// Rotation by a pure yaw quaternion (0,0,z,w): the general formula with x = y = 0 folded away.
struct Yaw {
  float s, wz2, zz2;  // 2w^2-1, 2wz, 2z^2
};
__device__ __forceinline__ Yaw make_yaw(Quat h) { return {2.0f * h.w * h.w - 1.0f, 2.0f * h.w * h.z, 2.0f * h.z * h.z}; }
__device__ __forceinline__ Vec3 yaw_rot(Yaw y, Vec3 v) {
  return {v.x * y.s - y.wz2 * v.y, v.y * y.s + y.wz2 * v.x, v.z * y.s + y.zz2 * v.z};
}

// (0,0,z,w) (x) q and q (x) (0,0,z,w): the Hamilton product with the zero components folded away
// (the reference multiplies by the heading quaternion with the general quat_mul; same value to ~1e-7).
__device__ __forceinline__ Quat yaw_mul_left(float z, float w, Quat q) {
  return {w * q.x - z * q.y, w * q.y + z * q.x, w * q.z + z * q.w, w * q.w - z * q.z};
}
__device__ __forceinline__ Quat yaw_mul_right(Quat q, float z, float w) {
  return {q.x * w + q.y * z, q.y * w - q.x * z, q.w * z + q.z * w, q.w * w - q.z * z};
}

// phc/utils/torch_utils.py:100-113 (quat_to_tan_norm): rotated x axis, then rotated z axis.
__device__ __forceinline__ void qsix(Quat q, float* o) {
  float s = 2.0f * q.w * q.w - 1.0f;
  float w2 = 2.0f * q.w;
  // rot(q, [1,0,0]): v*s + cross(qv, v)*2w + qv*(2 qv.v);  cross(qv,[1,0,0]) = (0, q.z, -q.y)
  float dx = 2.0f * q.x;
  o[0] = s + q.x * dx;
  o[1] = q.z * w2 + q.y * dx;
  o[2] = -q.y * w2 + q.z * dx;
  // rot(q, [0,0,1]): cross(qv,[0,0,1]) = (q.y, -q.x, 0)
  float dz = 2.0f * q.z;
  o[3] = q.y * w2 + q.x * dz;
  o[4] = -q.x * w2 + q.y * dz;
  o[5] = s + q.z * dz;
}

// isaacgym.torch_utils.normalize_angle [3P-memory]: atan2(sin x, cos x) -- general argument.
__device__ __forceinline__ float wrap_angle(float x) { return atan2f(sinf(x), cosf(x)); }

// The same function restricted to x = 2*acos(w) in [0, 2*pi]: identity below pi, x - 2*pi from
// fp32(pi) upwards (sin(fp32(pi)) < 0, so the reference maps fp32(pi) itself to -pi).  Differs from
// the atan2 form by < 5e-7.
__device__ __forceinline__ float wrap_angle_0_2pi(float x) { return x >= 3.14159274f ? x - 6.28318548f : x; }

// a / b with the hardware reciprocal (2 ulp); only for quantities under the 1e-4 float tolerance.
__device__ __forceinline__ float fdiv_fast(float a, float b) { return __fdividef(a, b); }

// sin(x) for x in [0, pi/2] (slerp arguments are (1-t)*h and t*h with h <= pi/2): odd Taylor
// polynomial through x^15, truncation error < 1e-9, no range reduction, no slow path.
__device__ __forceinline__ float sin_0_halfpi(float x) {
  const float z = x * x;
  float p = -7.6471637e-13f;           // -1/15!
  p = fmaf(p, z, 1.6059044e-10f);      //  1/13!
  p = fmaf(p, z, -2.5052108e-8f);      // -1/11!
  p = fmaf(p, z, 2.7557319e-6f);       //  1/9!
  p = fmaf(p, z, -1.9841270e-4f);      // -1/7!
  p = fmaf(p, z, 8.3333333e-3f);       //  1/5!
  p = fmaf(p, z, -1.6666667e-1f);      // -1/3!
  return fmaf(x * z, p, x);
}

// phc/utils/torch_utils.py:57-78 (quat_to_angle_axis): angle only (used by the rotation reward).
__device__ __forceinline__ float quat_angle(Quat q) {
  float s = sqrtf(1.0f - q.w * q.w);
  float ang = wrap_angle_0_2pi(2.0f * acosf(q.w));
  return (fabsf(s) > 1e-5f) ? ang : 0.0f;  // NaN s (|w|>1) fails the test like the reference's mask
}

// phc/utils/torch_utils.py:81-97 (quat_to_exp_map)
__device__ __forceinline__ Vec3 quat_exp_map(Quat q) {
  float s = sqrtf(1.0f - q.w * q.w);
  float ang = wrap_angle_0_2pi(2.0f * acosf(q.w));
  if (!(fabsf(s) > 1e-5f)) return {0.0f, 0.0f, 0.0f};  // angle 0 * default axis
  const float k = fdiv_fast(ang, s);
  return {k * q.x, k * q.y, k * q.z};
}

// isaacgym.torch_utils.quat_from_angle_axis with axis = +z [3P-memory], incl. the final quat_unit.
__device__ __forceinline__ Quat yaw_quat(float angle) {
  float s, c;
  sincosf(angle * 0.5f, &s, &c);
  float n = fmaxf(sqrtf(s * s + c * c), 1e-9f);
  return {0.0f, 0.0f, s / n, c / n};
}

// phc/utils/torch_utils.py:148-172 (exp_map_to_quat)
__device__ __forceinline__ Quat exp_map_quat(Vec3 e) {
  float ang = sqrtf(fmaf(e.z, e.z, fmaf(e.y, e.y, e.x * e.x)));
  Vec3 axis = {e.x / ang, e.y / ang, e.z / ang};
  ang = wrap_angle(ang);
  if (!(fabsf(ang) > 1e-5f)) {
    ang = 0.0f;
    axis = {0.0f, 0.0f, 1.0f};
  }
  float an = fmaxf(sqrtf(fmaf(axis.z, axis.z, fmaf(axis.y, axis.y, axis.x * axis.x))), 1e-9f);
  float s, c;
  sincosf(ang * 0.5f, &s, &c);
  Quat q = {axis.x / an * s, axis.y / an * s, axis.z / an * s, c};
  float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-9f);
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}

// phc/utils/torch_utils.py:175-197 (slerp); result is NOT renormalised, as in the reference.
__device__ __forceinline__ Quat slerp(Quat a, Quat b, float t) {
  float c = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  if (c < 0.0f) {
    b = {-b.x, -b.y, -b.z, -b.w};
  }
  c = fabsf(c);
  if (c >= 1.0f) return a;
  // 1 - c*c cancels badly near c = 1: keep the reference's two roundings (an FMA here would be MORE
  // accurate than the reference and move the result by up to ~3e-4 relative at small angles)
  float s = sqrtf(__fsub_rn(1.0f, __fmul_rn(c, c)));
  if (fabsf(s) < 0.001f) {
    return {0.5f * a.x + 0.5f * b.x, 0.5f * a.y + 0.5f * b.y, 0.5f * a.z + 0.5f * b.z, 0.5f * a.w + 0.5f * b.w};
  }
  const float h = acosf(c);
  const float inv_s = fdiv_fast(1.0f, s);
  const float ra = sin_0_halfpi((1.0f - t) * h) * inv_s;
  const float rb = sin_0_halfpi(t * h) * inv_s;
  return {ra * a.x + rb * b.x, ra * a.y + rb * b.y, ra * a.z + rb * b.z, ra * a.w + rb * b.w};
}

// phc/utils/torch_utils.py:200-212 (calc_heading)
__device__ __forceinline__ float heading_angle(Quat q) {
  float s = 2.0f * q.w * q.w - 1.0f;
  float rx = s + 2.0f * q.x * q.x;
  float ry = 2.0f * q.w * q.z + 2.0f * q.x * q.y;
  return atan2f(ry, rx);
}

// calc_heading_quat / calc_heading_quat_inv (torch_utils.py:215-240) without the angle round trip:
// from the rotated x axis (rx, ry) the half-angle sine / cosine follow algebraically, so no atan2 /
// sincos is needed.  heading = atan2(ry, rx); returns (sin(h/2), cos(h/2)); h_fwd = (0,0,s,c),
// h_inv = (0,0,-s,c).  Agrees with the angle form to ~2e-7 (the reference's final quat_unit included).
__device__ __forceinline__ void heading_half(Quat q, float& s_half, float& c_half) {
  const float s = 2.0f * q.w * q.w - 1.0f;
  const float rx = s + 2.0f * q.x * q.x;
  const float ry = 2.0f * q.w * q.z + 2.0f * q.x * q.y;
  const float n2 = rx * rx + ry * ry;
  if (!(n2 > 0.0f)) {  // atan2(0, 0) = 0
    s_half = 0.0f;
    c_half = 1.0f;
    return;
  }
  const float inv = rsqrtf(n2);
  const float ch = rx * inv, sh = ry * inv;
  if (ch >= 0.0f) {
    c_half = sqrtf(0.5f * (1.0f + ch));
    s_half = fdiv_fast(0.5f * sh, c_half);
  } else {
    s_half = copysignf(sqrtf(0.5f * (1.0f - ch)), sh);
    c_half = fdiv_fast(0.5f * sh, s_half);
  }
}

// ---- exact-order pieces (their results decide integer outputs) ---------------------------------

// (1-b)*p0 + b*p1 [+ off]: motion_lib_base.py:476-479, each product / sum rounded separately.
__device__ __forceinline__ float lerp_rn(float p0, float p1, float b) {
  return __fadd_rn(__fmul_rn(__fsub_rn(1.0f, b), p0), __fmul_rn(b, p1));
}

// torch.norm(d, dim=-1) on CPU for a length-3 row == sqrt(fma(z,z, fma(y,y, x*x))) (measured).
__device__ __forceinline__ float norm3_rn(float x, float y, float z) {
  return __fsqrt_rn(__fmaf_rn(z, z, __fmaf_rn(y, y, __fmul_rn(x, x))));
}

// motion time: progress(int64)*dt + start + offset, three fp32 roundings (humanoid_im.py:732,859,1120)
__device__ __forceinline__ float motion_time_rn(long long progress, float dt, float start, float off) {
  return __fadd_rn(__fadd_rn(__fmul_rn(__ll2float_rn(progress), dt), start), off);
}

// motion_lib_base.py:546-556 (_calc_frame_blend), bit-exact index arithmetic.
__device__ __forceinline__ void frame_blend_rn(float time, float len, long long nf, float mdt, long long& i0,
                                               long long& i1, float& blend) {
  float phase = __fdiv_rn(time, len);
  phase = fminf(fmaxf(phase, 0.0f), 1.0f);
  if (time < 0.0f) time = 0.0f;
  i0 = (long long)__fmul_rn(phase, __ll2float_rn(nf - 1));
  i1 = min(i0 + 1, nf - 1);
  float b = __fdiv_rn(__fsub_rn(time, __fmul_rn(__ll2float_rn(i0), mdt)), mdt);
  blend = fminf(fmaxf(b, 0.0f), 1.0f);
}

}  // namespace pulse
