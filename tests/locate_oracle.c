/* locate_oracle.c — CPU restatement of the geometry queries' point location (f2b_locate_points, DESIGN.md §3i).
 *
 * TEST INFRASTRUCTURE ONLY (tests/locate_oracle.py builds and binds it).  No reference counterpart: the reference renders images
 * only.  The oracle's own TreeNode / TransInfo layouts and warp_point (QueryFrameTransform in the march's roundings) are
 * reused by including oracle/f2_oracle.c; compiled, like it, with -ffp-contract=off so the only fused operations are fmaf(). */
#include "../oracle/f2_oracle.c"

/* The leaf holding each point by a walk from the root over half-open cubes [c - s/2, c + s/2), child slot
 * (x >= cx) << 2 | (y >= cy) << 1 | (z >= cz) (ConstructTreeNode, PersSampler.cpp:359-421), every visited node's own cube tested
 * (compacted trees skip levels), at most MAX_STACK levels like the march; then the point warped by the leaf's TransInfo.
 * anchors [n,2] = (trans_idx, leaf); (-1, -1) and warped 0 where the point is outside, in a dead child slot or in a leaf with
 * trans_idx < 0. */
void orc_locate_points(const void* tree_nodes, const void* trans_v, const float* pts, int n, float* warped, int* anchors) {
  const TreeNode* nodes = (const TreeNode*)tree_nodes;
  const TransInfo* trans = (const TransInfo*)trans_v;
  for (int i = 0; i < n; i++) {
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    int u = 0, leaf = -1;
    for (int depth = 0; depth < MAX_STACK; depth++) {
      const TreeNode* nd = nodes + u;
      const float hf = nd->side_len * .5f, cx = nd->center[0], cy = nd->center[1], cz = nd->center[2];
      if (!(x >= cx - hf && x < cx + hf && y >= cy - hf && y < cy + hf && z >= cz - hf && z < cz + hf)) break;
      int live = 0;
      for (int k = 0; k < 8; k++) live |= nd->childs[k] >= 0;
      if (!live) { if (nd->trans_idx >= 0) leaf = u; break; }
      const int v = nd->childs[((x >= cx) << 2) | ((y >= cy) << 1) | (z >= cz)];
      if (v < 0) break;
      u = v;
    }
    float* w = warped + 3 * (size_t)i;
    w[0] = w[1] = w[2] = 0.f;
    anchors[2 * (size_t)i] = -1; anchors[2 * (size_t)i + 1] = -1;
    if (leaf >= 0) {
      warp_point(trans + nodes[leaf].trans_idx, x, y, z, w);
      anchors[2 * (size_t)i] = nodes[leaf].trans_idx; anchors[2 * (size_t)i + 1] = leaf;
    }
  }
}
