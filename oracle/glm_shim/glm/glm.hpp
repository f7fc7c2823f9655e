// Minimal stand-in for the subset of g-truc/glm that the reference rasterizer uses.
//
// TEST INFRASTRUCTURE ONLY.  The reference checkout pins glm as an un-vendored submodule
// (g-truc/glm @ 6f14f4792a0cde5d0cf2c910506724d61cb95834, the reference's .SUBMODULES.json) and the
// directory third_party/glm is empty, so the reference CUDA sources cannot be compiled without
// something that answers `#include <glm/glm.hpp>`.  This header is written from scratch for that one
// purpose (oracle/build_ref.py).  It is never included by the product kernels.
//
// Semantics mirrored from glm's published behaviour:
//   * matrices are column-major: m[c] is column c, m[c][r] is row r of column c;
//   * mat3(a,b,c, d,e,f, g,h,i) fills column 0 with (a,b,c), column 1 with (d,e,f), ...;
//   * mat3(s) is s * identity;
//   * (A*B)[c][r] = A[0][r]*B[c][0] + A[1][r]*B[c][1] + A[2][r]*B[c][2]  (left to right);
//   * (A*v)[r]    = A[0][r]*v[0]   + A[1][r]*v[1]   + A[2][r]*v[2];
//   * dot(a,b) = a.x*b.x + a.y*b.y + a.z*b.z, length = sqrt(dot), normalize = v * inversesqrt(dot);
//   * outerProduct(c, r)[i] = c * r[i].
// "The reference" for bit-exact key parity therefore means: reference sources + this header, built by
// the same nvcc as the product (see DESIGN.md, section Oracle).
#pragma once
#include <cmath>
#include <cuda_runtime.h>

#define GLM_FN __host__ __device__ __forceinline__

namespace glm {

typedef int length_t;
enum qualifier { packed_highp, defaultp = packed_highp };

template <length_t L, typename T, qualifier Q = defaultp> struct vec;
template <length_t C, length_t R, typename T, qualifier Q = defaultp> struct mat;

template <typename T, qualifier Q> struct vec<2, T, Q> {
	T x, y;
	GLM_FN vec() : x(0), y(0) {}
	GLM_FN vec(T a, T b) : x(a), y(b) {}
	GLM_FN T& operator[](length_t i) { return (&x)[i]; }
	GLM_FN const T& operator[](length_t i) const { return (&x)[i]; }
};

template <typename T, qualifier Q> struct vec<3, T, Q> {
	T x, y, z;
	GLM_FN vec() : x(0), y(0), z(0) {}
	GLM_FN explicit vec(T s) : x(s), y(s), z(s) {}
	template <typename A, typename B, typename C>
	GLM_FN vec(A a, B b, C c) : x(T(a)), y(T(b)), z(T(c)) {}
	GLM_FN T& operator[](length_t i) { return (&x)[i]; }
	GLM_FN const T& operator[](length_t i) const { return (&x)[i]; }
	GLM_FN vec& operator+=(const vec& o) { x += o.x; y += o.y; z += o.z; return *this; }
	GLM_FN vec& operator+=(T s) { x += s; y += s; z += s; return *this; }
	GLM_FN vec& operator-=(const vec& o) { x -= o.x; y -= o.y; z -= o.z; return *this; }
	GLM_FN vec& operator*=(T s) { x *= s; y *= s; z *= s; return *this; }
	GLM_FN vec& operator/=(T s) { x /= s; y /= s; z /= s; return *this; }
};

template <typename T, qualifier Q> struct vec<4, T, Q> {
	T x, y, z, w;
	GLM_FN vec() : x(0), y(0), z(0), w(0) {}
	GLM_FN vec(T a, T b, T c, T d) : x(a), y(b), z(c), w(d) {}
	GLM_FN T& operator[](length_t i) { return (&x)[i]; }
	GLM_FN const T& operator[](length_t i) const { return (&x)[i]; }
};

typedef vec<2, float, defaultp> vec2;
typedef vec<3, float, defaultp> vec3;
typedef vec<4, float, defaultp> vec4;

// ---- vec3 arithmetic ------------------------------------------------------------------------------
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator+(const vec<3, T, Q>& a, const vec<3, T, Q>& b) { return vec<3, T, Q>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator-(const vec<3, T, Q>& a, const vec<3, T, Q>& b) { return vec<3, T, Q>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator-(const vec<3, T, Q>& a) { return vec<3, T, Q>(-a.x, -a.y, -a.z); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator*(const vec<3, T, Q>& a, const vec<3, T, Q>& b) { return vec<3, T, Q>(a.x * b.x, a.y * b.y, a.z * b.z); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator*(const vec<3, T, Q>& a, T s) { return vec<3, T, Q>(a.x * s, a.y * s, a.z * s); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator*(T s, const vec<3, T, Q>& a) { return vec<3, T, Q>(s * a.x, s * a.y, s * a.z); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator/(const vec<3, T, Q>& a, T s) { return vec<3, T, Q>(a.x / s, a.y / s, a.z / s); }
// float-vec3 mixed with int / double scalars (the reference writes `2 * v`, `v * 0.5`-style expressions)
GLM_FN vec3 operator*(int s, const vec3& a) { return float(s) * a; }
GLM_FN vec3 operator*(const vec3& a, int s) { return a * float(s); }
GLM_FN vec3 operator*(double s, const vec3& a) { return float(s) * a; }
GLM_FN vec3 operator*(const vec3& a, double s) { return a * float(s); }
GLM_FN vec3 operator/(const vec3& a, int s) { return a / float(s); }
GLM_FN vec3 operator/(const vec3& a, double s) { return a / float(s); }

// ---- vec2 arithmetic (only construction / member access is used, keep a few for safety) ------------
template <typename T, qualifier Q> GLM_FN vec<2, T, Q> operator+(const vec<2, T, Q>& a, const vec<2, T, Q>& b) { return vec<2, T, Q>(a.x + b.x, a.y + b.y); }
template <typename T, qualifier Q> GLM_FN vec<2, T, Q> operator*(const vec<2, T, Q>& a, T s) { return vec<2, T, Q>(a.x * s, a.y * s); }

// ---- vec4 arithmetic ------------------------------------------------------------------------------
template <typename T, qualifier Q> GLM_FN vec<4, T, Q> operator*(const vec<4, T, Q>& a, T s) { return vec<4, T, Q>(a.x * s, a.y * s, a.z * s, a.w * s); }
template <typename T, qualifier Q> GLM_FN vec<4, T, Q> operator/(const vec<4, T, Q>& a, T s) { return vec<4, T, Q>(a.x / s, a.y / s, a.z / s, a.w / s); }

// ---- scalar helpers -------------------------------------------------------------------------------
GLM_FN float abs(float v) { return ::fabsf(v); }
GLM_FN double abs(double v) { return ::fabs(v); }
GLM_FN int abs(int v) { return v < 0 ? -v : v; }
GLM_FN float sqrt(float v) { return ::sqrtf(v); }
GLM_FN double sqrt(double v) { return ::sqrt(v); }
GLM_FN float max(float a, float b) { return a < b ? b : a; }
GLM_FN float min(float a, float b) { return b < a ? b : a; }
GLM_FN float inversesqrt(float v) { return 1.0f / ::sqrtf(v); }

template <typename T, qualifier Q> GLM_FN vec<3, T, Q> max(const vec<3, T, Q>& a, T s) { return vec<3, T, Q>(max(a.x, s), max(a.y, s), max(a.z, s)); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> abs(const vec<3, T, Q>& a) { return vec<3, T, Q>(abs(a.x), abs(a.y), abs(a.z)); }

template <typename T, qualifier Q> GLM_FN T dot(const vec<3, T, Q>& a, const vec<3, T, Q>& b) {
	vec<3, T, Q> tmp(a * b);
	return tmp.x + tmp.y + tmp.z;
}
template <typename T, qualifier Q> GLM_FN T dot(const vec<4, T, Q>& a, const vec<4, T, Q>& b) {
	return (a.x * b.x + a.y * b.y) + (a.z * b.z + a.w * b.w);
}
template <typename T, qualifier Q> GLM_FN T dot(const vec<2, T, Q>& a, const vec<2, T, Q>& b) { return a.x * b.x + a.y * b.y; }
template <length_t L, typename T, qualifier Q> GLM_FN T length(const vec<L, T, Q>& a) { return sqrt(dot(a, a)); }
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> normalize(const vec<3, T, Q>& a) { return a * inversesqrt(dot(a, a)); }
template <typename T, qualifier Q> GLM_FN vec<4, T, Q> normalize(const vec<4, T, Q>& a) { return a * inversesqrt(dot(a, a)); }

// ---- mat3 -----------------------------------------------------------------------------------------
template <typename T, qualifier Q> struct mat<3, 3, T, Q> {
	typedef vec<3, T, Q> col_type;
	col_type c[3];
	GLM_FN mat() {}
	GLM_FN explicit mat(T s) { c[0] = col_type(s, 0, 0); c[1] = col_type(0, s, 0); c[2] = col_type(0, 0, s); }
	template <typename A0, typename A1, typename A2, typename B0, typename B1, typename B2, typename C0, typename C1, typename C2>
	GLM_FN mat(A0 x0, A1 y0, A2 z0, B0 x1, B1 y1, B2 z1, C0 x2, C1 y2, C2 z2) {
		c[0] = col_type(x0, y0, z0); c[1] = col_type(x1, y1, z1); c[2] = col_type(x2, y2, z2);
	}
	GLM_FN col_type& operator[](length_t i) { return c[i]; }
	GLM_FN const col_type& operator[](length_t i) const { return c[i]; }
	GLM_FN mat& operator+=(const mat& o) { c[0] += o.c[0]; c[1] += o.c[1]; c[2] += o.c[2]; return *this; }
};
typedef mat<3, 3, float, defaultp> mat3;

template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> transpose(const mat<3, 3, T, Q>& m) {
	return mat<3, 3, T, Q>(m[0][0], m[1][0], m[2][0], m[0][1], m[1][1], m[2][1], m[0][2], m[1][2], m[2][2]);
}
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator*(const mat<3, 3, T, Q>& a, const mat<3, 3, T, Q>& b) {
	mat<3, 3, T, Q> r;
	for (int col = 0; col < 3; col++)
		for (int row = 0; row < 3; row++)
			r[col][row] = a[0][row] * b[col][0] + a[1][row] * b[col][1] + a[2][row] * b[col][2];
	return r;
}
template <typename T, qualifier Q> GLM_FN vec<3, T, Q> operator*(const mat<3, 3, T, Q>& m, const vec<3, T, Q>& v) {
	return vec<3, T, Q>(
		m[0][0] * v.x + m[1][0] * v.y + m[2][0] * v.z,
		m[0][1] * v.x + m[1][1] * v.y + m[2][1] * v.z,
		m[0][2] * v.x + m[1][2] * v.y + m[2][2] * v.z);
}
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator*(const mat<3, 3, T, Q>& m, T s) { mat<3, 3, T, Q> r; r[0] = m[0] * s; r[1] = m[1] * s; r[2] = m[2] * s; return r; }
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator*(T s, const mat<3, 3, T, Q>& m) { mat<3, 3, T, Q> r; r[0] = m[0] * s; r[1] = m[1] * s; r[2] = m[2] * s; return r; }
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator/(const mat<3, 3, T, Q>& m, T s) { mat<3, 3, T, Q> r; r[0] = m[0] / s; r[1] = m[1] / s; r[2] = m[2] / s; return r; }
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator+(const mat<3, 3, T, Q>& a, const mat<3, 3, T, Q>& b) { mat<3, 3, T, Q> r; r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; return r; }
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator-(const mat<3, 3, T, Q>& a, const mat<3, 3, T, Q>& b) { mat<3, 3, T, Q> r; r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2]; return r; }
template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> operator-(const mat<3, 3, T, Q>& a) { mat<3, 3, T, Q> r; r[0] = -a[0]; r[1] = -a[1]; r[2] = -a[2]; return r; }
GLM_FN mat3 operator*(int s, const mat3& m) { return float(s) * m; }
GLM_FN mat3 operator*(double s, const mat3& m) { return float(s) * m; }

template <typename T, qualifier Q> GLM_FN mat<3, 3, T, Q> outerProduct(const vec<3, T, Q>& col, const vec<3, T, Q>& row) {
	mat<3, 3, T, Q> r;
	r[0] = col * row[0]; r[1] = col * row[1]; r[2] = col * row[2];
	return r;
}

}  // namespace glm
