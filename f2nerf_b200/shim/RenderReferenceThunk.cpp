// RenderReferenceThunk.cpp — compiled with -DRender=RenderReference, like the reference's own Renderer.cpp in the
// drop-in build (oracle/Makefile.ref, INTEGRATION.md section 3): under that macro the class declaration in
// Renderer/Renderer.h names the reference's body `RenderReference`, and this one-line wrapper makes it callable from
// B200Renderer.cpp (which sees the header without the macro) — used when F2B_RENDER=reference selects the reference path.
#include "Renderer/Renderer.h"

RenderResult f2b_reference_render(Renderer* r, const torch::Tensor& rays_o, const torch::Tensor& rays_d, const torch::Tensor& bounds,
                                  const torch::Tensor& emb_idx) {
  return r->Render(rays_o, rays_d, bounds, emb_idx);      // expands to r->RenderReference(...)
}
