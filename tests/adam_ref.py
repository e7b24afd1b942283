"""Float64 reference of gsb_adam_step (DESIGN.md section 12): the activations of the raw parameters, the chain rule of the
activated records' gradient back to them, and torch.optim.Adam's update (no weight decay) restated with torch's own tensor
operations, per learning-rate group.  Test infrastructure only."""
import torch

# learning-rate groups of gsb_adam_config.lr, in order, and their columns of the 60-float record
GROUPS = {"position": slice(0, 3), "scale": slice(4, 7), "opacity": slice(7, 8), "rotation": slice(8, 12),
          "sh_dc": slice(12, 15), "sh_rest": slice(15, 60)}


def _f64(a):
    return torch.as_tensor(a).to(torch.float64)


def activate(params):
    """The activated records of raw parameters: (p, 1), exp(log s), sigmoid(logit), q / |q|, SH."""
    p = _f64(params)
    v = p.clone()
    v[:, 3] = 1.0
    v[:, 4:7] = p[:, 4:7].exp()
    v[:, 7] = torch.sigmoid(p[:, 7])
    v[:, 8:12] = p[:, 8:12] / p[:, 8:12].norm(dim=1, keepdim=True)
    return v


def chain(params, grad_vertices):
    """dL/d(raw parameters) from dL/d(activated record): d log s = ds s, d logit = do o (1 - o),
    d q = (d q^ - q^ (q^ . d q^)) / |q|, position and SH unchanged; column 3 is 0."""
    p, g = _f64(params), _f64(grad_vertices)
    out = g.clone()
    out[:, 3] = 0.0
    out[:, 4:7] = g[:, 4:7] * p[:, 4:7].exp()
    o = torch.sigmoid(p[:, 7])
    out[:, 7] = g[:, 7] * o * (1 - o)
    n = p[:, 8:12].norm(dim=1, keepdim=True)
    qh = p[:, 8:12] / n
    dqh = g[:, 8:12]
    out[:, 8:12] = (dqh - qh * (qh * dqh).sum(1, keepdim=True)) / n
    return out


def adam_update(params, exp_avg, exp_avg_sq, grad, lr, beta1, beta2, eps, bias_correction1, bias_correction2_sqrt, rows=None):
    """torch.optim.Adam's step (foreach=False, no weight decay) with the given bias corrections, group by group on contiguous
    copies (the layout torch's Adam sees for a per-group parameter), over `rows` (a bool mask or index; None = every row).
    Returns the new (params, exp_avg, exp_avg_sq) as float64 tensors; the other rows and column 3 are unchanged."""
    P, M, V, G = (_f64(t).clone() for t in (params, exp_avg, exp_avg_sq, grad))
    sel = slice(None) if rows is None else torch.as_tensor(rows)
    for k, (name, cols) in enumerate(GROUPS.items()):
        x, m, v, g = (T[sel, cols].contiguous() for T in (P, M, V, G))
        # torch/optim/adam.py, _single_tensor_adam
        m.lerp_(g, 1 - beta1)
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        step_size = lr[k] / bias_correction1
        denom = (v.sqrt() / bias_correction2_sqrt).add_(eps)
        x.addcdiv_(m, denom, value=-step_size)
        for T, t in ((P, x), (M, m), (V, v)):
            T[sel, cols] = t
    return P, M, V


def step(params, exp_avg, exp_avg_sq, grad_vertices, cfg, rows=None):
    """One gsb_adam_step with gsb_adam_config `cfg` (its fp32 values): (params, exp_avg, exp_avg_sq, vertices), float64."""
    P, M, V = adam_update(params, exp_avg, exp_avg_sq, chain(params, grad_vertices), list(cfg.lr), cfg.beta1, cfg.beta2, cfg.eps,
                          cfg.bias_correction1, cfg.bias_correction2_sqrt, rows)
    return P, M, V, activate(P)
