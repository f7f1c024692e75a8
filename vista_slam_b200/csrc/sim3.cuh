// The Sim(3) algebra of the device pose graph (slam_graph.cu), in the [t | q | s] layout of PyPose (tx ty tz | qx qy qz
// qw | s): the product of keyframe insertion and node replay, the rotation -> quaternion of an edge measurement and the
// quaternion -> 4x4 of the export.  Every kernel that composes or prints a pose goes through these, so two paths that
// compose the same inputs in the same order agree bit for bit.
#pragma once

namespace sta {
namespace {

// Sim(3) a * b in the [t | q | s] layout; the quaternion is kept with w >= 0.
__device__ void sim3_mul(const float* a, const float* b, float* o) {
  const float ax = a[3], ay = a[4], az = a[5], aw = a[6];
  const float bx = b[3], by = b[4], bz = b[5], bw = b[6];
  // t = t_a + s_a R_a t_b, with R_a t_b = t_b + 2 w (u x t_b) + 2 u x (u x t_b)
  const float tx = b[0], ty = b[1], tz = b[2];
  const float cx = ay * tz - az * ty, cy = az * tx - ax * tz, cz = ax * ty - ay * tx;
  const float rx = tx + 2.f * (aw * cx + ay * cz - az * cy);
  const float ry = ty + 2.f * (aw * cy + az * cx - ax * cz);
  const float rz = tz + 2.f * (aw * cz + ax * cy - ay * cx);
  float q[4] = {aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz};
  const float sg = q[3] < 0.f ? -1.f : 1.f;
  o[0] = a[0] + a[7] * rx;
  o[1] = a[1] + a[7] * ry;
  o[2] = a[2] + a[7] * rz;
  for (int i = 0; i < 4; ++i) o[3 + i] = sg * q[i];
  o[7] = a[7] * b[7];
}

// Rotation (row-major 3x3 inside a 4x4) -> unit quaternion (x, y, z, w), w >= 0 (Shepperd's method, fp64).
// Returns false when R is not orthonormal with det +1 to 1e-3 (what pp.mat2SE3(atol=1e-3) refuses).
__device__ bool rot_to_quat(const float* M, float* q) {
  double R[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r][c] = M[r * 4 + c];
  bool ok = true;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double d = R[r][0] * R[c][0] + R[r][1] * R[c][1] + R[r][2] * R[c][2] - (r == c ? 1.0 : 0.0);
      ok = ok && fabs(d) <= 1e-3;
    }
  const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                     R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
  ok = ok && fabs(det - 1.0) <= 1e-3;
  double x[4];
  const double t = R[0][0] + R[1][1] + R[2][2];
  if (t > 0) {
    const double s = sqrt(t + 1.0) * 2;
    x[0] = (R[2][1] - R[1][2]) / s; x[1] = (R[0][2] - R[2][0]) / s; x[2] = (R[1][0] - R[0][1]) / s; x[3] = 0.25 * s;
  } else {
    int i = 0;
    if (R[1][1] > R[i][i]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    const double s = sqrt(1.0 + R[i][i] - R[j][j] - R[k][k]) * 2;
    x[i] = 0.25 * s;
    x[j] = (R[j][i] + R[i][j]) / s;
    x[k] = (R[k][i] + R[i][k]) / s;
    x[3] = (R[k][j] - R[j][k]) / s;
  }
  const double sg = x[3] < 0 ? -1.0 : 1.0;
  const double nrm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3]);
  for (int e = 0; e < 4; ++e) q[e] = static_cast<float>(sg * x[e] / nrm);
  return ok;
}

// The 4x4 pose of a Sim(3) p with the scale dropped: LieTensor.rotation().matrix() (the quaternion is not normalised)
// and the translation; returns the scale.
__device__ float sim3_to_pose44(const float* p, float* P) {
  const float x = p[3], y = p[4], z = p[5], w = p[6];
  const float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) P[r * 4 + c] = R[r * 3 + c];
    P[r * 4 + 3] = p[r];
  }
  P[12] = 0.f; P[13] = 0.f; P[14] = 0.f; P[15] = 1.f;
  return p[7];
}

}  // namespace
}  // namespace sta
