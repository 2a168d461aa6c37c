"""The OptNet QP layer with its parameterisation fused in (SURVEY 8f.3, example-cls-layer.ipynb:107-130):

    Q = tril(L) tril(L)^T + eps I,   h = G z0 + s0        (L, G, z0, s0: shared nn.Parameters)
    z = QPFunction(verbose=-1)(Q, p, G, h, e, e)          (p: the batched output of the previous layer)

`OptNetQP(eps)(L, G, z0, s0, p)` is that block as ONE autograd.Function: one launch builds Q and h
(`qpb200_optnet_construct`), pre_factor_kkt + the PDIPM kernel solve the batch with a single shared system, the
backward kernel reduces the per-sample gradients of the shared Q, G, h to their batch MEAN on the fly (qp.py:159-177:
no (B, nz, nz) tensor ever exists) and one launch maps them onto the parameters (`qpb200_optnet_chain`): dL, dG, dz0,
ds0. The notebook's version runs ~8 torch kernels with (nz, nz) temporaries before and after every QPFunction call and
materialises nothing different; results are identical to composing the same formulas with torch autograd around
`qpth_b200.QPFunction` (tests/test_gpu_layers.py).

Only the lower triangle of L is read: its strictly upper triangle may hold anything, NaN included, the results are those
of tril(L), and the gradient dL is exactly zero above the diagonal. The Q built from it reaches the QP kernels, which
read only its lower triangle."""
import torch

from . import _lib
from ._lib import ptr
from .qp import solve_forward, solve_backward


def OptNetQP(eps=1e-4, qp_eps=1e-12, notImprovedLim=3, maxIter=20):
    class OptNetQPFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, L, G, z0, s0, p):
            assert L.is_cuda and L.dtype == torch.float64, "OptNetQP: fp64 CUDA tensors"
            n, m = L.size(0), G.size(0)
            lib = _lib.load()
            Lc, Gc, z0c, s0c = (t.detach().contiguous() for t in (L, G, z0, s0))
            Q = torch.empty(n, n, dtype=torch.float64, device=L.device)
            h = torch.empty(m, dtype=torch.float64, device=L.device)
            with torch.cuda.device(L.device):
                _lib.check(lib.qpb200_optnet_construct(n, m, ptr(Lc), ptr(Gc), ptr(z0c), ptr(s0c), float(eps), ptr(Q),
                                                       ptr(h), _lib.stream()))
            e = torch.empty(0, dtype=torch.float64, device=L.device)
            st = solve_forward(Q, p.detach(), Gc, h, e, e, eps=qp_eps, verbose=-1, notImprovedLim=notImprovedLim,
                               maxIter=maxIter, check_Q_spd=False)
            ctx.st, ctx.saved = st, (Lc, Gc, z0c)
            return st.zhat.clone()

        @staticmethod
        def backward(ctx, dl_dz):
            Lc, Gc, z0c = ctx.saved
            n, m = Lc.size(0), Gc.size(0)
            lib = _lib.load()
            dQ, dp, dGq, dh, _, _ = solve_backward(ctx.st, dl_dz, [True, False, True, True, True, True],
                                                   [True, True, True, True, False, False])
            f64 = dict(dtype=torch.float64, device=Lc.device)
            dL = torch.empty(n, n, **f64); dG = torch.empty(m, n, **f64); dz0 = torch.empty(n, **f64); ds0 = torch.empty(m, **f64)
            with torch.cuda.device(Lc.device):
                _lib.check(lib.qpb200_optnet_chain(n, m, ptr(Lc), ptr(Gc), ptr(z0c), ptr(dQ), ptr(dGq), ptr(dh),
                                                   ptr(dL), ptr(dG), ptr(dz0), ptr(ds0), _lib.stream()))
            return dL, dG, dz0, ds0, dp

    return OptNetQPFn.apply
