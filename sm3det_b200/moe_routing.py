"""Gating of the MoE layers, shared by functional.MoEBlockFn, lsk_functional.MoELinearFn and expert_parallel.EPMoEBlockFn.

The only caller of the router, plan, assign and router-backward entry points: the gating noise, one routing forward
(router -> plan -> assign) into a `Routing` record, the routing state each Function saves for its backward, and the router
backward.  Nothing here reads a device value on the host: the step is captured in a CUDA graph.
"""
import torch

from . import ops
from .ops import EPI_RESID

# what the router saves for its backward (the noisy-gating ones are None under clean gating)
_ROUTER_SAVES = ('logits', 'p', 'sigma', 'top_vals', 'top_idx_m')


def gating_noise(layer, T, device):
    """[T, E] gating noise of a noisy-gating layer in training, else None.  Tests inject a fixed tensor as
    ``layer._injected_noise``; otherwise it is drawn on the device (one randn per layer and pass)."""
    if not (layer.noisy_gating and layer.training):
        return None
    noise = getattr(layer, '_injected_noise', None)
    if noise is None:
        noise = torch.randn((T, layer.num_experts), device=device, dtype=torch.float32)
    return noise.to(device, torch.float32).contiguous()


class Routing:
    """The routing of one MoE layer for one pass: the gate parameters and noise it was computed from, the top-k indices and
    gates, the pair space (`slot_of`, `pair_token`, the padded expert segments of the plan) and, when the router ran with
    save=True, its backward saves."""

    def __init__(self, **fields):
        self.__dict__.update(fields)

    @property
    def grouped(self):
        return self.tile_group, self.num_m_tiles

    @property
    def segs(self):
        return self.seg_begin, self.seg_end

    def record(self):
        """The routing fields of a layer's `record` entry (tests/parity_util.py reads them by these keys)."""
        return dict(top_idx=self.top_idx, top_gate=self.top_gate, importance=self.importance, load=self.load,
                    loss=self.loss, counts=self.counts)

    def save(self, ctx, *tensors, dispatch=True):
        """ctx.save_for_backward(*tensors, routing state).  dispatch=False leaves out the local pair list and segments
        (expert parallelism dispatches through its own exchange plan).  Without the router's saves (checkpointing), the
        projector bias is kept so that rerun_router can rebuild them."""
        names = ['wp', 'sim', 'tau', 'w_noise', 'noise', 'top_idx', 'top_gate', 'slot_of', 'importance', 'load']
        if dispatch:
            names += ['pair_token', 'seg_begin', 'seg_end', 'tile_group', 'num_m_tiles']
        names += list(_ROUTER_SAVES) if self.logits is not None else ['bp']
        ctx.save_for_backward(*tensors, *(getattr(self, n) for n in names))
        ctx.routing = (names, dict(E=self.E, k=self.k, rows=self.rows))

    @staticmethod
    def load(ctx):
        """Inverse of save: -> (the caller's tensors, Routing)."""
        names, meta = ctx.routing
        saved = ctx.saved_tensors
        n = len(saved) - len(names)
        return saved[:n], Routing(**dict(zip(names, saved[n:])), **meta)

    def rerun_router(self, v):
        """Checkpointed backward: rebuild the router's backward saves from the recomputed (bit-identical) v and the saved
        noise.  The routing and the plan stay the saved ones; nothing is re-planned."""
        T, C = v.shape
        r = ops.moe_router(v, self.wp, self.bp, self.sim, self.tau, T=T, Cc=C, E=self.E, k=self.k, w_noise=self.w_noise,
                           noise=self.noise, save=True)
        for n in _ROUTER_SAVES:
            setattr(self, n, r[n])


def route(v, wp, bp, sim, tau, w_noise, noise, E, k, save):
    """Router -> plan -> assign over the [T, C] router input v.  save: also keep what router_backward reads."""
    T, C = v.shape
    r = ops.moe_router(v, wp, bp, sim, tau, T=T, Cc=C, E=E, k=k, w_noise=w_noise, noise=noise, save=save)
    plan = ops.moe_plan(r['partials'], T=T, E=E, k=k)
    slot_of, pair_token = ops.moe_assign(r['top_idx'], plan, T=T, E=E, k=k)
    return Routing(E=E, k=k, rows=plan['max_rows'], wp=wp, bp=bp, sim=sim, tau=tau, w_noise=w_noise, noise=noise,
                   top_idx=r['top_idx'], top_gate=r['top_gate'], slot_of=slot_of, pair_token=pair_token,
                   **{n: plan[n] for n in ('importance', 'load', 'loss', 'counts', 'seg_begin', 'seg_end', 'tile_group',
                                           'num_m_tiles')},
                   **{n: r[n] for n in _ROUTER_SAVES})


def router_backward(rt, v, dgate, dloss, wp_t=None):
    """Backward of the gating from the gate gradient dgate [T, k] and the gate-loss gradient dloss.
    -> (dv_r [T, C] router contribution to dv, dwp, dbp, dsim, dtau, dw_noise).  wp_t: packed image of wp for the dgrad.
    dw_noise is None when the layer has no w_noise and zero when it ran without noise."""
    T, C = v.shape
    E, k = rt.E, rt.k
    P = rt.wp.shape[0]
    dev = v.device
    dtau = torch.zeros((1,), device=dev, dtype=torch.float32)
    dsim = torch.zeros((P, E), device=dev, dtype=torch.float32)
    lscale = dloss.reshape(1).contiguous().float()
    noisy = rt.noise is not None          # gates depend on w_noise whenever noise was added, also for k == E
    nz = dict(noise=rt.noise, sigma=rt.sigma, top_vals=rt.top_vals, top_idx_m=rt.top_idx_m, load=rt.load) if noisy else None
    dp, dr = ops.moe_router_bwd(rt.p, rt.sim, rt.tau, rt.top_idx, rt.top_gate, dgate, rt.logits, rt.importance, lscale,
                                dsim, dtau, T=T, E=E, k=k, noisy=nz)
    dwp = torch.zeros_like(rt.wp)
    ops.linear_wgrad(dp, v, dwp)
    dbp = torch.zeros((P,), device=dev, dtype=torch.float32)
    ops.colsum(dp, dbp, rows=T, Cc=P)
    dv_r = ops.linear_dgrad(dp, rt.wp, packed=wp_t)
    dwn = None
    if noisy:
        # r = v @ w_noise is an [T,C]x[C,E] product with E < 32: run it as a 32-wide zero-padded GEMM pair
        wn_t = torch.zeros((32, C), device=dev, dtype=torch.float32)
        wn_t[:E] = rt.w_noise.t()
        dwn_t = torch.zeros((32, C), device=dev, dtype=torch.float32)
        ops.linear_wgrad(dr, v, dwn_t)                             # [32,C] = dr^T v
        dwn = dwn_t[:E].t().contiguous()
        dv_r = ops.linear_dgrad(dr, wn_t, epilogue=EPI_RESID, resid=dv_r)
    elif rt.w_noise is not None:
        dwn = torch.zeros((C, E), device=dev, dtype=torch.float32)
    return dv_r, dwp, dbp, dsim, dtau, dwn
