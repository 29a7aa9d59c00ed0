// B200Renderer.h — run-time switches of the fused Renderer::Render body (B200Renderer.cpp).
#pragma once
// true: Render also fills Renderer::sample_result_ in the reference's compact layout (one extra scan + gather; the trainer
// never reads it, debug dumps do).  Default: env F2B_KEEP_SAMPLES=1.
void f2b_render_keep_samples(bool on);
// true: route Renderer::Render to the reference's own body (compiled as RenderReference).  Default: env F2B_RENDER=reference.
void f2b_render_use_reference(bool on);
// How many TRAIN backwards so far reused the kept table-gradient storage (zero-filling its live prefix) and how many
// allocated a fresh, fully zeroed one (first step, or a trainer still holding last step's gradient).
void f2b_render_grad_storage_counts(long* reused, long* fresh);
