"""Native target descriptors.

The reference takes an opaque Python ``log_prob_func`` (samplers.py:857-858) and differentiates it with
autograd (samplers.py:65).  An opaque callable cannot enter a CUDA kernel, so the engine recognises a
small family of *descriptors*.  Every descriptor is

* a valid reference ``log_prob_func`` (``__call__`` takes a 1-D tensor, returns a scalar, is written with plain
  torch ops) -- the *same object* drives the oracle / the unmodified reference and the CUDA kernels; and
* a description of the analytic gradient the kernels evaluate, with the fp32 operation order chosen so that
  ``torch.autograd.grad(self(x), x)`` and the in-kernel gradient agree bit for bit (``grad`` restates that
  order in torch ops; tests/test_targets.py pins the equality on CPU).

Anything else passed as ``log_prob_func`` is refused by ``hamiltorch_b200.sample`` with a clear error: there
is no CPU fallback on the product path.
"""
import math

import torch

# target kinds -- must match include/hmcx.h
KIND_GAUSS_ISO = 0
KIND_GAUSS_DIAG = 1
KIND_GAUSS_FULL = 2
KIND_FUNNEL = 3
KIND_MLP = 4

_LOG_2PI = math.log(2.0 * math.pi)


class Target:
    """Base class: a log-density the sm_90a kernels know how to differentiate."""

    kind = -1
    dim = 0

    def __call__(self, x):  # pragma: no cover - abstract
        raise NotImplementedError

    def grad(self, x):  # pragma: no cover - abstract
        raise NotImplementedError

    def _tensors(self):
        return {}

    def to(self, device):
        """Return a copy of the descriptor whose parameter tensors live on ``device``."""
        import copy
        new = copy.copy(self)
        for name, t in self._tensors().items():
            setattr(new, name, t.to(device))
        return new


class GaussianIso(Target):
    """log p(x) = -0.5 * sum(x*x)  (+ -0.5*D*log(2*pi) when ``normalized``).

    BASELINE config 2 / 5 target (SURVEY.md section 8d).  Gradient: -x (exact in fp32).
    """

    kind = KIND_GAUSS_ISO

    def __init__(self, dim, normalized=False):
        self.dim = int(dim)
        self.log_norm = float(-0.5 * self.dim * _LOG_2PI) if normalized else 0.0

    def __call__(self, x):
        lp = -0.5 * (x * x).sum()
        if self.log_norm != 0.0:
            lp = lp + self.log_norm
        return lp

    def grad(self, x):
        return -x


class GaussianDiag(Target):
    """Independent Gaussian, log p(x) = -0.5 * sum((x-mean)^2 * inv_var) + log_norm.

    BASELINE config 1 (the notebook's diag-covariance 3-D Gaussian, notebooks/hamiltorch_log_prob_examples.ipynb
    cell 6) and the reference's own reversibility test target (tests/test_util.py:98-101).
    fp32 op order (shared with the kernel): y = x-mean; g = -(inv_var*y).
    """

    kind = KIND_GAUSS_DIAG

    def __init__(self, mean, var, normalized=True):
        mean = torch.as_tensor(mean, dtype=torch.float32).flatten().clone()
        var = torch.as_tensor(var, dtype=torch.float32).flatten().clone()
        if mean.shape != var.shape:
            raise ValueError('mean and var must have the same length')
        self.dim = mean.numel()
        self.mean = mean
        self.inv_var = 1.0 / var
        if normalized:
            self.log_norm = float(-0.5 * (self.dim * _LOG_2PI + torch.log(var.double()).sum().item()))
        else:
            self.log_norm = 0.0

    def _tensors(self):
        return {'mean': self.mean, 'inv_var': self.inv_var}

    def __call__(self, x):
        y = x - self.mean
        lp = -0.5 * ((y * y) * self.inv_var).sum()
        if self.log_norm != 0.0:
            lp = lp + self.log_norm
        return lp

    def grad(self, x):
        return -(self.inv_var * (x - self.mean))


class GaussianFull(Target):
    """Correlated Gaussian with precision matrix P: log p(x) = -0.5 * y.(P y) + log_norm, y = x-mean.

    P is symmetrised at construction.  Gradient (kernel order): g = -(P y) with the row dot products
    accumulated in fp32.
    """

    kind = KIND_GAUSS_FULL

    def __init__(self, mean, cov=None, prec=None, normalized=True):
        mean = torch.as_tensor(mean, dtype=torch.float32).flatten().clone()
        if (cov is None) == (prec is None):
            raise ValueError('give exactly one of cov / prec')
        if prec is None:
            prec = torch.linalg.inv(torch.as_tensor(cov, dtype=torch.float64))
        prec = torch.as_tensor(prec, dtype=torch.float64)
        prec = 0.5 * (prec + prec.t())
        self.dim = mean.numel()
        if prec.shape != (self.dim, self.dim):
            raise ValueError('precision must be (D, D)')
        self.mean = mean
        self.prec = prec.to(torch.float32).contiguous()
        if normalized:
            self.log_norm = float(-0.5 * (self.dim * _LOG_2PI - torch.linalg.slogdet(prec)[1].item()))
        else:
            self.log_norm = 0.0

    def _tensors(self):
        return {'mean': self.mean, 'prec': self.prec}

    def __call__(self, x):
        y = x - self.mean
        lp = -0.5 * torch.dot(y, torch.mv(self.prec, y))
        if self.log_norm != 0.0:
            lp = lp + self.log_norm
        return lp

    def grad(self, x):
        return -torch.mv(self.prec, x - self.mean)


class Funnel(Target):
    """Neal's funnel as in notebooks/hamiltorch_log_prob_examples.ipynb cell 22:
    v = w[0] ~ N(0, sigma_v^2),  w[1:] ~ N(0, exp(-v)).

    Closed form (SURVEY.md section 8d cfg 3; avoids torch.distributions' scale validation, section 8a quirks):
      log p = -v^2/(2 sigma_v^2) - 0.5*log(2 pi sigma_v^2) + n*(0.5*v - 0.5*log 2pi) - 0.5*exp(v)*sum(x^2)
    """

    kind = KIND_FUNNEL

    def __init__(self, dim, sigma_v=3.0):
        if dim < 2:
            raise ValueError('funnel needs dim >= 2')
        self.dim = int(dim)
        self.sigma_v = float(sigma_v)
        self.inv_var_v = 1.0 / (self.sigma_v ** 2)
        n = self.dim - 1
        self.log_norm = float(-0.5 * math.log(2.0 * math.pi * self.sigma_v ** 2) - 0.5 * n * _LOG_2PI)

    def __call__(self, w):
        v = w[0]
        x = w[1:]
        n = self.dim - 1
        return (-0.5 * self.inv_var_v) * (v * v) + (0.5 * n) * v - 0.5 * torch.exp(v) * (x * x).sum() + self.log_norm

    def grad(self, w):
        v = w[0]
        x = w[1:]
        n = self.dim - 1
        ev = torch.exp(v)
        gv = -(self.inv_var_v * v) + 0.5 * n - 0.5 * ev * (x * x).sum()
        gx = -(ev * x)
        return torch.cat([gv.reshape(1), gx])


def is_target(obj):
    return isinstance(obj, Target)


# ----------------------------------------------------------------------------------------------------------
# Bayesian MLP: the log_prob_func that define_model_log_prob builds (samplers.py:1093-1201)
# ----------------------------------------------------------------------------------------------------------
ACT_NONE, ACT_RELU, ACT_TANH, ACT_SIGMOID = 0, 1, 2, 3
_ACT_OF_MODULE = {'ReLU': ACT_RELU, 'Tanh': ACT_TANH, 'Sigmoid': ACT_SIGMOID}
# model_loss (samplers.py:1170-1184) -> kernel loss id (include/hmcx.h HMCX_LOSS_*)
LOSS_REGRESSION, LOSS_BINARY, LOSS_MULTICLASS, LOSS_MULTICLASS_LOGSOFTMAX = 0, 1, 2, 3
LOSS_ID = {'regression': LOSS_REGRESSION, 'binary_class_linear_output': LOSS_BINARY,
           'multi_class_linear_output': LOSS_MULTICLASS, 'multi_class_log_softmax_output': LOSS_MULTICLASS_LOGSOFTMAX}
MLP_MAX_LAYERS = 8


def mlp_spec(model):
    """Recognise a dense stack: ``nn.Linear`` or ``nn.Sequential(Linear, [ReLU|Tanh|Sigmoid], Linear, ...
    [, LogSoftmax])`` with biases.  Returns (widths [n_0..n_L], activations [after layer l], Linear modules,
    final_log_softmax).  Anything else -- conv / recurrent / normalisation layers, or a module whose forward() is
    arbitrary Python -- cannot be turned into a CUDA kernel the way util.make_functional (util.py:253-376) turns it
    into a closure, and is refused."""
    import torch.nn as nn
    mods = [model] if isinstance(model, nn.Linear) else (list(model) if isinstance(model, nn.Sequential) else None)
    if mods is None:
        raise NotImplementedError(
            'hamiltorch_b200 runs Bayesian-NN sampling for dense stacks only: pass an nn.Sequential of '
            'Linear / ReLU / Tanh / Sigmoid layers (got %s)' % type(model).__name__)
    final_log_softmax = False
    if mods and isinstance(mods[-1], nn.LogSoftmax):
        if mods[-1].dim not in (1, -1):
            raise NotImplementedError('LogSoftmax must act on the class dimension (dim=1)')
        final_log_softmax = True
        mods = mods[:-1]
    widths, acts, linears = [], [], []
    for m in mods:
        if isinstance(m, nn.Linear):
            if m.bias is None:
                raise NotImplementedError('Linear layers without bias are not supported')
            if widths and widths[-1] != m.in_features:
                raise ValueError('layer widths do not chain')
            if not widths:
                widths.append(m.in_features)
            widths.append(m.out_features)
            acts.append(ACT_NONE)
            linears.append(m)
        elif type(m).__name__ in _ACT_OF_MODULE:
            if not linears or acts[-1] != ACT_NONE:
                raise NotImplementedError('an activation must follow a Linear layer')
            acts[-1] = _ACT_OF_MODULE[type(m).__name__]
        else:
            raise NotImplementedError('unsupported layer for the dense-stack kernel: %s' % type(m).__name__)
    if not linears:
        raise NotImplementedError('no Linear layer found')
    if acts[-1] != ACT_NONE:
        raise NotImplementedError('the model must end with a Linear layer (optionally followed by LogSoftmax)')
    if len(linears) > MLP_MAX_LAYERS:
        raise NotImplementedError('at most %d Linear layers' % MLP_MAX_LAYERS)
    return widths, acts, linears, final_log_softmax


def _act(h, a):
    if a == ACT_RELU:
        return torch.relu(h)
    if a == ACT_TANH:
        return torch.tanh(h)
    if a == ACT_SIGMOID:
        return torch.sigmoid(h)
    return h


class MLPTarget(Target):
    """log p(theta) = ll + prior/prior_scale for a dense stack -- the closure define_model_log_prob builds:

        prior = sum over parameter tensors i of Normal(0, tau_i^-1/2).log_prob(w_i).sum()   (samplers.py:1141-1157)
        ll    = 'regression'                     -0.5*tau_out*((f(x)-y)**2).sum(0)                        (:1184)
                'binary_class_linear_output'     -tau_out*BCEWithLogitsLoss(sum)(f(x), y)                  (:1170-1172)
                'multi_class_linear_output'      -tau_out*CrossEntropyLoss(sum)(f(x), y.long().view(-1))   (:1173-1177)
                'multi_class_log_softmax_output' -tau_out*nll_loss(f(x), y.long().view(-1))  [mean!]       (:1179-1180)

    ``theta`` is the flat vector in ``model.parameters()`` order, each tensor row-major (util.py:121-136): for every
    Linear the (out, in) weight then the (out,) bias.  ``__call__`` restates the reference's closure with the same
    torch ops, so it is also a valid reference ``log_prob_func`` (regression returns shape (O,) -- (1,) for a scalar
    output, SURVEY 8a quirk; the classification losses return a 0-d tensor).  ``x is None`` samples the prior.
    """

    kind = KIND_MLP
    predict_mode = False       # define_model_log_prob(predict=True): the closure also returns the network output

    def __init__(self, widths, acts, x, y, tau_list, tau_out=1., prior_scale=1.0, model_loss='regression',
                 final_log_softmax=False):
        if model_loss not in LOSS_ID:
            raise NotImplementedError(
                'model_loss %r has no CUDA kernel (callable losses cannot enter a kernel); supported: %s'
                % (model_loss, sorted(LOSS_ID)))
        self.model_loss = model_loss
        self.loss_id = LOSS_ID[model_loss]
        self.final_log_softmax = bool(final_log_softmax)
        if self.final_log_softmax != (model_loss == 'multi_class_log_softmax_output'):
            raise NotImplementedError("a LogSoftmax output layer goes with model_loss='multi_class_log_softmax_output' "
                                      "(and only with it)")
        self.widths = list(widths)
        self.acts = list(acts)
        self.num_layers = len(self.widths) - 1
        self.dim = sum(self.widths[l] * self.widths[l + 1] + self.widths[l + 1] for l in range(self.num_layers))
        self.x = None if x is None else x.detach().to(torch.float32)
        self.y = None if y is None else y.detach().to(torch.float32)
        self.y_cols = self.widths[-1] if self.loss_id in (LOSS_REGRESSION, LOSS_BINARY) else 1
        if self.x is not None:
            if self.x.dim() != 2 or self.x.shape[1] != self.widths[0]:
                raise ValueError('x must be (N, %d)' % self.widths[0])
            if self.y.numel() != self.x.shape[0] * self.y_cols:
                raise ValueError('y must have %d entries per data point for %s' % (self.y_cols, model_loss))
        self.tau_out = float(tau_out)
        self.prior_scale = prior_scale
        tau_list = [torch.as_tensor(t, dtype=torch.float32) for t in tau_list]
        if len(tau_list) != 2 * self.num_layers:
            raise ValueError('tau_list needs one precision per parameter tensor (%d)' % (2 * self.num_layers))
        self.tau_list = tau_list
        self.sizes = []
        for l in range(self.num_layers):
            self.sizes += [self.widths[l] * self.widths[l + 1], self.widths[l + 1]]
        # constants with the reference's fp32 roundings (torch.distributions.Normal.log_prob)
        self.scale = [t ** -0.5 for t in tau_list]                       # samplers.py:1143
        self.two_var = [2 * (s ** 2) for s in self.scale]
        self.log_scale = [s.log() for s in self.scale]
        self.grad_coef = [(torch.tensor(1.0) / prior_scale) / tv for tv in self.two_var]   # see DESIGN.md 3.4

    @classmethod
    def from_model(cls, model, x, y, tau_list=None, tau_out=1., prior_scale=1.0, model_loss='regression'):
        widths, acts, linears, fls = mlp_spec(model)
        if tau_list is None:
            tau_list = [torch.tensor(1.)] * (2 * len(linears))           # samplers.py:1348-1355
        return cls(widths, acts, x, y, tau_list, tau_out, prior_scale, model_loss, fls)

    def _tensors(self):
        d = {}
        if self.x is not None:
            d['x'], d['y'] = self.x, self.y
        return d

    def unflatten(self, params):
        out, i = [], 0
        for l in range(self.num_layers):
            n_in, n_out = self.widths[l], self.widths[l + 1]
            W = params[i:i + n_in * n_out].view(n_out, n_in)
            i += n_in * n_out
            b = params[i:i + n_out]
            i += n_out
            out.append((W, b))
        return out

    def forward(self, params, x):
        h = x
        for l, (W, b) in enumerate(self.unflatten(params)):
            h = _act(torch.nn.functional.linear(h, W, b), self.acts[l])
        if self.final_log_softmax:
            h = torch.nn.functional.log_softmax(h, dim=1)
        return h

    def log_prior(self, params):
        i = 0
        l_prior = torch.zeros_like(params[0])
        for n, s in zip(self.sizes, self.scale):
            w = params[i:i + n]
            l_prior = torch.distributions.Normal(torch.zeros_like(s), s, validate_args=False).log_prob(w).sum() + l_prior
            i += n
        return l_prior

    def __call__(self, params, predict=None):
        predict = self.predict_mode if predict is None else predict
        l_prior = self.log_prior(params)
        if self.x is None:
            return l_prior / self.prior_scale
        output = self.forward(params, self.x.to(params.device))
        y = self.y.to(params.device)
        if self.loss_id == LOSS_BINARY:
            ll = - self.tau_out * torch.nn.BCEWithLogitsLoss(reduction='sum')(output, y.view_as(output))
        elif self.loss_id == LOSS_MULTICLASS:
            ll = - self.tau_out * torch.nn.CrossEntropyLoss(reduction='sum')(output, y.long().view(-1))
        elif self.loss_id == LOSS_MULTICLASS_LOGSOFTMAX:
            ll = - self.tau_out * torch.nn.functional.nll_loss(output, y.long().view(-1))
        else:
            ll = - 0.5 * self.tau_out * ((output - y.view_as(output)) ** 2).sum(0)
        if predict:
            return (ll + l_prior / self.prior_scale), output
        return ll + l_prior / self.prior_scale

    def grad(self, params):
        p = params.detach().requires_grad_()
        return torch.autograd.grad(self(p), p)[0]


MLPRegression = MLPTarget      # the regression-only name used by round-1 callers
