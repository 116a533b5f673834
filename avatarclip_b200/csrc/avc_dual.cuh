// avc_dual.cuh -- forward-mode dual numbers for the rotation chains of avc_motion.cu (pytorch3d's 6D -> axis-angle)
// and avc_pose.cu (VPoser's Gram-Schmidt -> torchgeometry matrot2aa).  A chain written once as a template on its scalar
// type S gives its values with S = float and one column of its Jacobian with S = Dual (the input's tangent set to a unit
// vector), so the value and its derivative come from one definition.  Every branch is taken on the value, as autograd
// does.
#pragma once

namespace avc {

struct Dual {
  float v, d;
};
__device__ __forceinline__ Dual operator+(Dual a, Dual b) { return {a.v + b.v, a.d + b.d}; }
__device__ __forceinline__ Dual operator-(Dual a, Dual b) { return {a.v - b.v, a.d - b.d}; }
__device__ __forceinline__ Dual operator*(Dual a, Dual b) { return {a.v * b.v, a.d * b.v + a.v * b.d}; }
__device__ __forceinline__ Dual operator/(Dual a, Dual b) { return {a.v / b.v, (a.d * b.v - a.v * b.d) / (b.v * b.v)}; }
__device__ __forceinline__ Dual operator+(float a, Dual b) { return {a + b.v, b.d}; }
__device__ __forceinline__ Dual operator-(float a, Dual b) { return {a - b.v, -b.d}; }
__device__ __forceinline__ Dual operator*(float a, Dual b) { return {a * b.v, a * b.d}; }
__device__ __forceinline__ Dual operator*(Dual a, float b) { return {a.v * b, a.d * b}; }
__device__ __forceinline__ Dual operator/(Dual a, float b) { return {a.v / b, a.d / b}; }
__device__ __forceinline__ Dual operator/(float a, Dual b) { return {a / b.v, -a * b.d / (b.v * b.v)}; }
__device__ __forceinline__ Dual operator-(Dual a) { return {-a.v, -a.d}; }

__device__ __forceinline__ float val(float x) { return x; }
__device__ __forceinline__ float val(Dual x) { return x.v; }
template <class S> __device__ __forceinline__ S konst(float c);
template <> __device__ __forceinline__ float konst<float>(float c) { return c; }
template <> __device__ __forceinline__ Dual konst<Dual>(float c) { return {c, 0.f}; }
__device__ __forceinline__ float dsqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ Dual dsqrt(Dual x) { const float s = sqrtf(x.v); return {s, x.d / (2.f * s)}; }
__device__ __forceinline__ float dsin(float x) { return sinf(x); }
__device__ __forceinline__ Dual dsin(Dual x) { float s, c; sincosf(x.v, &s, &c); return {s, c * x.d}; }
__device__ __forceinline__ float dcos(float x) { return cosf(x); }
__device__ __forceinline__ Dual dcos(Dual x) { float s, c; sincosf(x.v, &s, &c); return {c, -s * x.d}; }
__device__ __forceinline__ float datan2(float y, float x) { return atan2f(y, x); }
__device__ __forceinline__ Dual datan2(Dual y, Dual x) {
  return {atan2f(y.v, x.v), (x.v * y.d - y.v * x.d) / (x.v * x.v + y.v * y.v)};
}

}  // namespace avc
