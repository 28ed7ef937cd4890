"""Vector fields the solver can fuse into its stage kernels.

`LinearField(weight)` is an ordinary `torch.nn.Module` with `forward(t, y) = y @ weight^T` (what `torch.nn.functional.linear`
computes), so it runs unchanged under the reference (`torchdiffeq.odeint(LinearField(W), y0, t)`).  Handed to
`torchdiffeq_b200.odeint` with an adaptive method, a float32 CUDA state `[..., 128]` and a `128 x 128` weight, every
Runge-Kutta stage -- the combination `y_i = y0 + sum_j coef_ij k_j` (rk_common.py:79) AND the evaluation `k_i = f(t_i, y_i)`
(rk_common.py:80) -- is ONE hand-written wgmma kernel (csrc/tdq_linear.cu): `y_i` never goes to memory, the float32
product runs on the tensor cores as a split-bfloat16 emulation (3 planes per operand, 6 products) with float32-grade accuracy.  Everything else about the solve (error
norm, controller, dense output, the device-side loop) is unchanged; `forward` itself is only called for f(t0, y0), the
initial step size and `jump_t` restarts.  With `options={'independent_rows': True}` (dopri5 / bosh3, `[B, 128]` rows, scalar
tolerances) every attempt of every row is one kernel with each row's own step (csrc/tdq_attempt.cu k_linear_rows_attempt);
the taped row solves of `differentiable` / `event_gradient` and `compact_rows` keep the generic row path.
`options={'fused_linear': False}` keeps the generic path (func as a torch call)."""
import torch


class LinearField(torch.nn.Module):
    """dy/dt = y @ weight^T.  weight: [D, D] tensor or Parameter (kept by reference: updates are picked up by the next solve)."""

    def __init__(self, weight, requires_grad=None):
        super().__init__()
        if weight.dim() != 2 or weight.shape[0] != weight.shape[1]:
            raise ValueError("LinearField needs a square [D, D] weight, got {}".format(tuple(weight.shape)))
        if isinstance(weight, torch.nn.Parameter) or requires_grad:
            self.weight = weight if isinstance(weight, torch.nn.Parameter) else torch.nn.Parameter(weight)
        else:
            self.register_buffer("weight", weight)

    def forward(self, t, y):
        return torch.nn.functional.linear(y, self.weight)


def fusable(func, shape, dtype, device, lib):
    """The weight tensor if func/state qualify for the fused stage kernel, else None."""
    if not isinstance(func, LinearField) or type(func).forward is not LinearField.forward:
        return None
    w = func.weight
    if (len(shape) < 1 or shape[-1] != w.shape[0] or dtype != torch.float32 or w.dtype != torch.float32
            or w.device != device or not w.is_contiguous() or w.data_ptr() % 16):
        return None
    if not lib.tdq_linear_supported(0, int(w.shape[0])):          # 0 = TDQ_F32
        return None
    return w
