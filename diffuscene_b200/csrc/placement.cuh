// Placement of a catalogue model at a generated object's pose, shared by scene evaluation (k_scene_boxes) and the
// renderer (render.cu), so both see the same world-space vertices bit for bit.
//
// scene_synthesis/utils.py:114-163 in its order: scale = size / raw_half, centroid = centre of the scaled raw AABB,
// v * scale - centroid, then .dot(R) + t with R[0][0] = R[2][2] = cos, R[0][2] = -sin, R[2][0] = sin built from the
// fp32 angle (np.cos of a float32 is a float32).  Every operation is an explicit _rn intrinsic in fp64.
#pragma once

namespace ds {

struct Placement {
  double kx, ky, kz;      // per-axis scale
  double cx, cy, cz;      // centre of the scaled raw AABB
  double c, s;            // float-rounded cos / sin of the angle
  double tx, ty, tz;      // translation
};

// size / trans: the object's 3 floats; raw_half [3] and raw_aabb [6] (min xyz, max xyz) of its model.
__device__ __forceinline__ Placement make_placement(const float* size, const float* trans, float angle,
                                                    const double* raw_half, const double* raw_aabb) {
  Placement p;
  p.kx = __ddiv_rn((double)size[0], raw_half[0]);
  p.ky = __ddiv_rn((double)size[1], raw_half[1]);
  p.kz = __ddiv_rn((double)size[2], raw_half[2]);
  p.cx = __dmul_rn(__dadd_rn(__dmul_rn(raw_aabb[0], p.kx), __dmul_rn(raw_aabb[3], p.kx)), 0.5);
  p.cy = __dmul_rn(__dadd_rn(__dmul_rn(raw_aabb[1], p.ky), __dmul_rn(raw_aabb[4], p.ky)), 0.5);
  p.cz = __dmul_rn(__dadd_rn(__dmul_rn(raw_aabb[2], p.kz), __dmul_rn(raw_aabb[5], p.kz)), 0.5);
  // correctly rounded float32 cos / sin of the float32 angle, as numpy's float32 cos / sin give them
  const double th = angle;
  p.c = __double2float_rn(cos(th));
  p.s = __double2float_rn(sin(th));
  p.tx = trans[0]; p.ty = trans[1]; p.tz = trans[2];
  return p;
}

// World x / z of an already scaled and centred point (px, pz): (px, ., pz) . R + t.
__device__ __forceinline__ void rotate_xz(const Placement& p, double px, double pz, double& x, double& z) {
  x = __dadd_rn(__dadd_rn(__dmul_rn(px, p.c), __dmul_rn(pz, p.s)), p.tx);
  z = __dadd_rn(__dadd_rn(__dmul_rn(px, -p.s), __dmul_rn(pz, p.c)), p.tz);
}

// World position of raw model vertex (vx, vy, vz).
__device__ __forceinline__ void place_vertex(const Placement& p, double vx, double vy, double vz, double& x, double& y,
                                             double& z) {
  rotate_xz(p, __dsub_rn(__dmul_rn(vx, p.kx), p.cx), __dsub_rn(__dmul_rn(vz, p.kz), p.cz), x, z);
  y = __dadd_rn(__dsub_rn(__dmul_rn(vy, p.ky), p.cy), p.ty);
}

}  // namespace ds
