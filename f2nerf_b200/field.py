"""Hash3DAnchored + TCNNWP — host-side mirrors of the reference's field operators
(``src/Field/Hash3DAnchored.{h,cpp,cu}``, ``src/Field/TCNNWP.{h,cpp}``) over the C ABI.

State tensors keep the reference's names, dtypes and shapes so reference checkpoints load
(``Hash3DAnchored::States``, Hash3DAnchored.cpp:112-122): ``feat_pool_`` fp32 [pool,2] (leaf),
``prim_pool_`` i32 [16,V,3], ``bias_pool_`` f32 [16*V,3], ``mlp_.params_`` fp32 (leaf).
"""
import math

import numpy as np
import torch

from . import ops
from .rng import burn_mlp_output

N_LEVELS, N_CHANNELS = 16, 2
LOSS_SCALE = 128.0


def tcnn_xavier_params(d_in, n_hidden_layers, seed=19970826):
    """tiny-cuda-nn's initialize_xavier_uniform driven by pcg32 (gpu_matrix.h:291-306,
    dependencies/pcg32/pcg32.h:57-116, TCNNWP.cpp:96-97) — host-side, runs once at construction."""
    mask = (1 << 64) - 1
    state, inc = 0, (1 << 1) | 1

    def nxt():
        nonlocal state
        old = state
        state = (old * 0x5851f42d4c957f2d + inc) & mask
        xs = (((old >> 18) ^ old) >> 27) & 0xffffffff
        rot = old >> 59
        return ((xs >> rot) | (xs << ((-rot) & 31))) & 0xffffffff

    nxt(); state = (state + seed) & mask; nxt()
    mats = [(64, d_in)] + [(64, 64)] * (n_hidden_layers - 1) + [(16, 64)]
    out = []
    for rows, cols in mats:
        scale = np.float32(math.sqrt(6.0 / (rows + cols)))
        u = np.array([(nxt() >> 9) | 0x3f800000 for _ in range(rows * cols)], dtype=np.uint32).view(np.float32)
        out.append((u - np.float32(1.0)) * np.float32(2.0) * scale - scale)
    return torch.from_numpy(np.concatenate(out).astype(np.float32))


class TCNNWP:
    """TCNNWP (TCNNWP.h:11-35): FullyFusedMLP(d_in=32 -> 64 x n_hidden_layers -> 16 padded), no biases."""

    def __init__(self, global_data_pool, d_in, d_out, d_hidden, n_hidden_layers, device="cuda"):
        if d_in != 32 or d_hidden != 64 or d_out > 16 or n_hidden_layers not in (1, 2):
            raise NotImplementedError("TCNNWP(b200): only the shipped shapes 32 -> 64 x {1,2} -> <=16 are built")
        self.global_data_pool_ = global_data_pool
        self.d_in_, self.d_out_, self.d_hidden_, self.n_hidden_layers_ = d_in, d_out, d_hidden, n_hidden_layers
        self.loss_scale_ = LOSS_SCALE
        self.params_ = tcnn_xavier_params(d_in, n_hidden_layers).to(device).requires_grad_(True)

    @property
    def n_hidden_matmuls(self):
        return self.n_hidden_layers_ - 1

    def InitParams(self):
        self.params_.data.copy_(tcnn_xavier_params(self.d_in_, self.n_hidden_layers_))

    def params_f16(self):
        return ops.cast_f32_to_f16(self.params_.detach())

    def Query(self, pts):
        """TCNNWP::Query (TCNNWP.cpp:102-113): fp32 [n, 32] -> fp32 [n, d_out] (fp16-rounded values)."""
        return _MLPFunction.apply(pts.contiguous(), self.params_, self)[:, :self.d_out_].contiguous()


class _MLPFunction(torch.autograd.Function):
    """TCNNWPFunction (TCNNWP.cpp:117-243): loss-scaled fp16 backward, NaN back-off."""

    @staticmethod
    def forward(ctx, x, params, mlp):
        burn_mlp_output(x.shape[0], x.device)                    # TCNNWP.cpp:143: the reference's output is a torch::rand
        x16 = ops.cast_f32_to_f16(x)
        p16 = ops.cast_f32_to_f16(params)
        need = x.requires_grad or params.requires_grad
        out16, hidden = ops.mlp_fwd(x16, p16, mlp.n_hidden_matmuls, save_hidden=need)
        ctx.mlp = mlp
        ctx.saved = (x16, p16, hidden)
        return ops.cast_f16_to_f32(out16)

    @staticmethod
    def backward(ctx, g):
        mlp = ctx.mlp
        x16, p16, hidden = ctx.saved
        scale = mlp.loss_scale_
        d16 = ops.cast_f32_to_f16(g.contiguous(), scale)
        din16, dparams = ops.mlp_bwd(d16, x16, hidden, p16, mlp.n_hidden_matmuls, need_din=True)
        din = ops.cast_f16_to_f32(din16, 1.0 / scale)
        dparams = dparams / scale
        if not (torch.isfinite(din).all() and torch.isfinite(dparams).all()):
            mlp.global_data_pool_.backward_nan_ = True
            mlp.loss_scale_ = max(mlp.loss_scale_ / 2.0, 1.0)
        return din, dparams, None


def _is_prime(x):
    """Deterministic Miller-Rabin for x < 4 759 123 141 (bases 2, 7, 61); the reference trial-divides
    (Hash3DAnchored.cpp:39-44) — same predicate, the draws stay torch.randint(2^28, 2^30) on the CPU generator."""
    if x < 2:
        return False
    for q in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 61):
        if x % q == 0:
            return x == q
    d, r = x - 1, 0
    while d % 2 == 0:
        d //= 2; r += 1
    for a in (2, 7, 61):
        y = pow(a, d, x)
        if y in (1, x - 1):
            continue
        for _ in range(r - 1):
            y = y * y % x
            if y == x - 1:
                break
        else:
            return False
    return True


class Hash3DAnchored:
    """Hash3DAnchored (Hash3DAnchored.h:22-51)."""

    def __init__(self, global_data_pool, log2_table_size=19, mlp_hidden_dim=64, mlp_out_dim=16, n_hidden_layers=1,
                 rand_bias=True, device="cuda", prim_pool=None, bias_pool=None):
        self.global_data_pool_ = global_data_pool
        self.pool_size_ = (1 << log2_table_size) * N_LEVELS
        self.n_volumes_ = int(global_data_pool.n_volumes_)
        dev = torch.device(device)
        self.feat_pool_ = ((torch.rand((self.pool_size_, N_CHANNELS), dtype=torch.float32, device=dev) * .2 - 1.) * 1e-4)
        self.feat_pool_.requires_grad_(True)
        n = 3 * N_LEVELS * self.n_volumes_
        if prim_pool is None:
            prims = []                      # rejection-sampled primes in [2^28, 2^30): ONE int32 draw per trial on the CPU
            while len(prims) < n:           # generator, as Hash3DAnchored.cpp:49-55 does, so the generator is left in the same
                v = int(torch.randint(1 << 28, 1 << 30, (1,), dtype=torch.int32).item())   # state for the draws that follow
                if _is_prime(v):
                    prims.append(v)
            prim_pool = torch.tensor(prims[:n], dtype=torch.int32)
        self.prim_pool_ = torch.as_tensor(prim_pool, dtype=torch.int32).reshape(N_LEVELS, self.n_volumes_, 3).to(dev).contiguous()
        if bias_pool is None:
            bias_pool = (torch.rand((N_LEVELS * self.n_volumes_, 3), dtype=torch.float32, device=dev) * 1000. + 100.) \
                if rand_bias else torch.zeros((N_LEVELS * self.n_volumes_, 3), dtype=torch.float32, device=dev)
        self.bias_pool_ = torch.as_tensor(bias_pool, dtype=torch.float32).reshape(N_LEVELS * self.n_volumes_, 3).to(dev).contiguous()
        self.local_size_ = ((self.pool_size_ // N_LEVELS) >> 4) << 4        # Hash3DAnchored.cpp:73-75
        self.mlp_ = TCNNWP(global_data_pool, N_LEVELS * N_CHANNELS, mlp_out_dim, mlp_hidden_dim, n_hidden_layers, device)

    n_levels_ = N_LEVELS

    def table_f16(self):
        """fp16 shadow of the master table.  The reference re-casts all 64 MB on every call (Hash3DAnchored.cu:186);
        here the shadow is cached and reused while the master is unchanged: torch-side writes bump the tensor's
        version counter (-> re-cast), FusedAdam refreshes the shadow itself in the same kernel that updates the master."""
        if not getattr(self, "_shadow_managed_", False):          # default: like the reference, always from the master
            return ops.table_to_half(self.feat_pool_.detach())
        ver = self.feat_pool_._version
        sh = getattr(self, "_shadow_", None)
        if sh is None or self._shadow_ver_ != ver or sh.device != self.feat_pool_.device:
            sh = self._shadow_ = ops.table_to_half(self.feat_pool_.detach())
            self._shadow_ver_ = ver
        return sh

    def manage_shadow(self, on=True):
        """Opt in to the cached shadow (FusedAdam does).  While on, the master must only change through FusedAdam,
        ``Reset``/``LoadStates`` or version-tracked torch in-place ops (writes through ``.data`` are invisible to the cache)."""
        self._shadow_managed_ = bool(on)
        self._shadow_ = None

    def invalidate_shadow(self):
        self._shadow_ = None

    def shadow_for_update(self):
        """The fp16 shadow buffer a fused optimizer step writes next to the master (fully initialised first)."""
        return self.table_f16()

    def shadow_updated(self):
        self._shadow_ver_ = self.feat_pool_._version

    def AnchoredQuery(self, points, anchors):
        """Hash3DAnchored::AnchoredQuery (Hash3DAnchored.cpp:84-99): [n,3] warped points + [n] trans_idx
        -> fp32 [n, 16]; differentiable w.r.t. feat_pool_ and mlp_.params_."""
        return _FieldFunction.apply(self.feat_pool_, self.mlp_.params_, points.contiguous(), anchors.contiguous(), self)

    def States(self):
        return [self.feat_pool_.data, self.prim_pool_.data, self.bias_pool_.data,
                torch.full((1,), self.n_volumes_, dtype=torch.int32), self.mlp_.params_.data]

    def LoadStates(self, states, idx):
        self.feat_pool_.data.copy_(states[idx]); idx += 1
        self.invalidate_shadow()
        self.prim_pool_ = states[idx].clone().to(self.feat_pool_.device).contiguous(); idx += 1
        self.bias_pool_.data.copy_(states[idx]); idx += 1
        self.n_volumes_ = int(states[idx].item()); idx += 1
        self.mlp_.params_.data.copy_(states[idx]); idx += 1
        return idx

    def OptimParamGroups(self):
        lr = self.global_data_pool_.learning_rate_
        return [dict(params=[self.feat_pool_], lr=lr, betas=(0.9, 0.99), eps=1e-15),
                dict(params=[self.mlp_.params_], lr=lr, betas=(0.9, 0.99), eps=1e-15, weight_decay=1e-6)]

    def Reset(self):
        self.feat_pool_.data.uniform_(-1e-2, 1e-2)
        self.invalidate_shadow()
        self.mlp_.InitParams()


def field_forward(field, table16, params16, points, anchors, anchor_stride, save, logit_only=False, save_feat=None):
    """hash encode -> MLP.  Returns (out, feat16, hidden); out is fp32 [n,16], or [n] (channel 0) when
    ``logit_only``; feat16 when ``save`` or ``save_feat``, hidden only when ``save``.  For the default 32 -> 64 -> 16 field
    MLP this is ONE fused kernel (f2b_field_fwd); other depths run encode + MLP + cast."""
    save_feat = save if save_feat is None else save_feat
    if field.mlp_.n_hidden_matmuls == 0:
        return ops.field_fwd(table16, field.prim_pool_, field.bias_pool_, field.n_volumes_, field.local_size_, params16,
                             points, anchors, anchor_stride, logit_only=logit_only, save=save, save_feat=save_feat)
    feat16 = ops.hash_fwd(table16, field.prim_pool_, field.bias_pool_, field.n_volumes_, field.local_size_, points,
                          anchors, anchor_stride)
    out16, hidden = ops.mlp_fwd(feat16, params16, field.mlp_.n_hidden_matmuls, save_hidden=save and not logit_only)
    out = ops.cast_f16_to_f32(out16)
    if logit_only:
        out = out[:, 0].contiguous()
    return out, (feat16 if save_feat else None), hidden


def field_backward(field, params16, points, anchors, anchor_stride, feat16, hidden, d_out_f32):
    """dL/d out [n,16] fp32 -> (dL/d feat_pool fp32 [pool,2], dL/d mlp params fp32)."""
    scale = field.mlp_.loss_scale_
    d16 = ops.cast_f32_to_f16(d_out_f32, scale)
    dfeat16, dparams = ops.mlp_bwd(d16, feat16, hidden, params16, field.mlp_.n_hidden_matmuls, need_din=True)
    grad_table = torch.zeros_like(field.feat_pool_)
    ops.hash_bwd(field.prim_pool_, field.bias_pool_, field.n_volumes_, field.local_size_, points, anchors, anchor_stride, dfeat16,
                 1.0 / scale, grad_table)
    dparams = dparams / scale
    return grad_table, dparams


class _FieldFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat_pool, params, points, anchors, field):
        burn_mlp_output(points.shape[0], points.device)          # the MLP inside AnchoredQuery (TCNNWP.cpp:143)
        table16 = ops.table_to_half(feat_pool)
        params16 = ops.cast_f32_to_f16(params)
        need = feat_pool.requires_grad or params.requires_grad
        out, feat16, hidden = field_forward(field, table16, params16, points, anchors, 1, need)
        ctx.field = field
        ctx.saved = (params16, points, anchors, feat16, hidden)
        return out

    @staticmethod
    def backward(ctx, g):
        field = ctx.field
        params16, points, anchors, feat16, hidden = ctx.saved
        grad_table, dparams = field_backward(field, params16, points, anchors, 1, feat16, hidden, g.contiguous())
        if not torch.isfinite(dparams).all():
            field.global_data_pool_.backward_nan_ = True
            field.mlp_.loss_scale_ = max(field.mlp_.loss_scale_ / 2.0, 1.0)
        return grad_table, dparams, None, None, None
