/* normals_oracle.c — CPU restatement of the warp Jacobian the gradient kernel forms (warp_jacobian, DESIGN.md §3j).
 *
 * TEST INFRASTRUCTURE ONLY (tests/normals_oracle.py builds and binds it).  It includes tests/locate_oracle.c, and through it
 * oracle/f2_oracle.c, to reuse the point location, proj_xz and mix12 (the reference's QueryFrameTransformJac in its roundings,
 * as jac_dir_norm forms it); compiled, like them, with -ffp-contract=off so the only fused operations are fmaf(). */
#include "locate_oracle.c"

/* J [n,3,3] (row r = d warp_r / d x) at each point's leaf, PersSampler.cu:171-187; 0 where no valid leaf holds the point. */
void orc_warp_jacobian(const void* tree_nodes, const void* trans_v, const float* pts, int n, float* jac) {
  const TransInfo* trans = (const TransInfo*)trans_v;
  for (int i = 0; i < n; i++) {
    float w[3];
    int anc[2];
    orc_locate_points(tree_nodes, trans_v, pts + 3 * (size_t)i, 1, w, anc);
    float* J = jac + 9 * (size_t)i;
    for (int k = 0; k < 9; k++) J[k] = 0.f;
    if (anc[0] < 0) continue;
    const TransInfo* T = trans + anc[0];
    const float X = pts[3 * (size_t)i], Y = pts[3 * (size_t)i + 1], Z = pts[3 * (size_t)i + 2];
    float t0[12], t1[12], t2[12];
    for (int k = 0; k < 12; k++) {
      const float* a = T->w2xz[k];
      float xz0, xz1; proj_xz(a, X, Y, Z, &xz0, &xz1);
      const float r = 1.f / xz1;
      const float q = (-xz0) / (xz1 * xz1);
      t0[k] = fmaf(a[0], r, a[4] * q);
      t1[k] = fmaf(r, a[1], q * a[5]);
      t2[k] = fmaf(r, a[2], q * a[6]);
    }
    for (int r = 0; r < 3; r++) {
      J[3 * r] = mix12(T->weight[r], t0); J[3 * r + 1] = mix12(T->weight[r], t1); J[3 * r + 2] = mix12(T->weight[r], t2);
    }
  }
}
