"""Host-side driver of the sm_90a kernels: turns descriptors + torch tensors into C-ABI calls (include/hmcx.h).

Everything here is plumbing -- device buffers, padding to the (C, ld) layout, the step-size adaptation table,
the random-stream modes.  The arithmetic of the hot path lives in csrc/*.cu.
"""
import copy
import ctypes as C
import os
import math

import torch

from . import _native as N
from . import targets as T


# ----------------------------------------------------------------------------------------------------------
# descriptors -> native structs (tensors are kept alive on the wrapper object)
# ----------------------------------------------------------------------------------------------------------
def _combine_mlp_splits(splits):
    """A list of MLPRegression descriptors (what define_split_model_log_prob returns: one per data batch, sharing the
    network and the prior) -> (first descriptor, concatenated x, y, split_begin)."""
    first = splits[0]
    for d in splits:
        if not isinstance(d, T.MLPRegression):
            raise TypeError('a split log_prob_func list must hold MLPRegression descriptors')
        if d.widths != first.widths or d.acts != first.acts or d.tau_out != first.tau_out or \
                d.model_loss != first.model_loss or \
                float(d.prior_scale) != float(first.prior_scale) or \
                any(float(a) != float(b) for a, b in zip(d.tau_list, first.tau_list)):
            raise RuntimeError('all splits must share the network, tau_list, tau_out and prior_scale')
        if d.x is None:
            raise RuntimeError('split descriptors need data')
    x = torch.cat([d.x for d in splits])
    y = torch.cat([d.y.reshape(d.x.shape[0], first.y_cols) for d in splits])
    begin = [0]
    for d in splits:
        begin.append(begin[-1] + d.x.shape[0])
    return first, x, y, begin


def fold_targets(target, folds):
    """The K training sets of a K-fold run as a split list: split k is a copy of the MLPTarget ``target`` holding every
    data row i with ``folds[i] != k`` in the original order (rows with fold -1 are in every split), with the target's
    network, prior, prior_scale, tau_out and settings.  ``folds``: (N,) integers in -1 .. K-1, K = max + 1.

    Memory: the native form of the list (``NativeTarget``) concatenates the training sets, about (K - 1) N rows of x and
    y -- K N rows with reloo's -1 rows.  A tensor-core stack (n0 -> 128 -> nL) also packs x as 16 n0 bytes per row (tf32
    hi | lo in both GEMM layouts): once per training set, and once more for the all-rows tiling when a split boundary is
    not a multiple of 64 rows, i.e. up to 2 (K - 1) N rows of packed operand."""
    if not isinstance(target, T.MLPTarget) or target.x is None:
        raise TypeError('fold_targets: an MLPTarget with data')
    f = torch.as_tensor(folds).detach().to(device=target.x.device, dtype=torch.int64).reshape(-1)
    n = target.x.shape[0]
    if f.numel() != n:
        raise ValueError('fold_targets: folds has %d entries, the target has %d data rows' % (f.numel(), n))
    y = target.y.reshape(n, target.y_cols)
    out = []
    for k in range(int(f.max()) + 1):
        keep = f != k
        t = copy.copy(target)
        t.x, t.y = target.x[keep], y[keep]
        out.append(t)
    return out


class NativeTarget:
    def __init__(self, target, device):
        self.device = torch.device(device)
        self._keep = {}
        if isinstance(target, list) or isinstance(target, T.MLPRegression):
            self._init_mlp(target)
            return
        if not T.is_target(target):
            raise TypeError('not a hamiltorch_b200 target descriptor: %r' % (target,))
        self.target = target
        self.dim = target.dim
        self.num_splits = 1
        s = N.TargetStruct()
        s.kind, s.dim = target.kind, target.dim
        s.log_norm = float(getattr(target, 'log_norm', 0.0))
        for field, attr in (('mean', 'mean'), ('inv_var', 'inv_var'), ('prec', 'prec')):
            t = getattr(target, attr, None)
            if t is not None:
                t = t.detach().to(self.device, torch.float32).contiguous()
                self._keep[field] = t
                setattr(s, field, t.data_ptr())
        s.funnel_inv_var_v = float(getattr(target, 'inv_var_v', 0.0))
        self.struct = s

    def _init_mlp(self, target):
        if isinstance(target, list):
            first, x, y, begin = _combine_mlp_splits(target)
        else:
            first = target
            x = first.x
            y = None if x is None else first.y.reshape(x.shape[0], first.y_cols)
            begin = [0, 0 if x is None else x.shape[0]]
        if len(begin) - 1 > N.MLP_MAX_SPLITS:
            raise NotImplementedError('at most %d splits' % N.MLP_MAX_SPLITS)
        self.target = target
        self.dim = first.dim
        self.num_splits = len(begin) - 1
        self.mlp_desc = first
        m = N.MlpStruct()
        m.num_layers = first.num_layers
        for i, w in enumerate(first.widths):
            m.widths[i] = w
        for i, a in enumerate(first.acts):
            m.activation[i] = a
        m.loss = first.loss_id
        m.tau_out = first.tau_out
        m.prior_scale = float(first.prior_scale)
        for i in range(2 * first.num_layers):
            m.prior_two_var[i] = float(first.two_var[i])
            m.prior_log_scale[i] = float(first.log_scale[i])
            m.prior_grad_coef[i] = float(first.grad_coef[i])
        if x is not None:
            xd = x.detach().to(self.device, torch.float32).contiguous()
            yd = y.detach().to(self.device, torch.float32).contiguous()
            self._keep['x'], self._keep['y'] = xd, yd
            m.x, m.y = xd.data_ptr(), yd.data_ptr()
            m.num_rows = xd.shape[0]
        m.num_splits = self.num_splits
        m.cluster_size = int(getattr(first, 'cluster_size', 0))      # 0 = auto; 1/2/4 pins CTAs per chain
        m.tensor_cores = int(getattr(first, 'tensor_cores', 0))      # 0 = auto (tensor cores when the shape fits); 1 = off
        for i, b in enumerate(begin):
            m.split_begin[i] = b
        self.mlp_struct = m
        s = N.TargetStruct()
        s.kind, s.dim = T.KIND_MLP, first.dim
        s.mlp = C.pointer(m)
        self.struct = s
        if x is not None and m.tensor_cores == 0 and self.device.type == 'cuda':
            # tensor-core form: x as ready-made tensor-core operands (tf32 hi | lo, both GEMM layouts), built once per target
            lib = N.load_library()
            nbytes = int(lib.hmcx_mlp_packed_x_bytes(C.byref(s)))
            if nbytes:
                xp = torch.empty(nbytes // 4, dtype=torch.float32, device=self.device)
                with torch.cuda.device(self.device):
                    N.check(lib.hmcx_mlp_pack_x(C.byref(s), N.ptr(xp), N.stream_ptr(self.device)), 'hmcx_mlp_pack_x')
                self._keep['x_packed'] = xp
                m.x_packed = xp.data_ptr()

    def ref(self):
        return C.byref(self.struct)


# Descriptor targets (Gaussian / Funnel) carry small host tensors; uploading them is a pageable host-to-device copy = a host
# synchronisation per call.  The same descriptor object, unmodified, reuses its device operands (keyed like _MASS_CACHE; the
# entry holds the descriptor).  Bayesian-NN targets (lists / MLPRegression: data + packed operands) are rebuilt per call.
_TARGET_CACHE = []


def native_target(target, device):
    if isinstance(target, NativeTarget):
        return target
    if isinstance(target, list) or isinstance(target, T.MLPRegression) or not T.is_target(target):
        return NativeTarget(target, device)
    tensors = [t for t in (getattr(target, a, None) for a in ('mean', 'inv_var', 'prec')) if torch.is_tensor(t)]
    key = (id(target), tuple(id(t) for t in tensors), tuple(t._version for t in tensors), str(torch.device(device)),
           target.dim, float(getattr(target, 'log_norm', 0.0)), float(getattr(target, 'inv_var_v', 0.0)))
    for k, _, nt in _TARGET_CACHE:
        if k == key:
            return nt
    nt = NativeTarget(target, device)
    _TARGET_CACHE.append((key, target, nt))
    if len(_TARGET_CACHE) > 8:
        _TARGET_CACHE.pop(0)
    return nt


class NativeMass:
    """inv_mass as the reference accepts it (None | (D,) | (D,D)); the mass used by gibbs is inverted ONCE with
    the same torch ops as samplers.py:942-952 so that sqrt(mass) is bit-identical."""

    def __init__(self, inv_mass, dim, device):
        self.device = torch.device(device)
        s = N.MassStruct()
        self._keep = {}
        if inv_mass is None:
            s.kind = N.MASS_NONE
        elif isinstance(inv_mass, list):
            # block list (samplers.py:188-197, :287-292, :803-809, :944-947) == the block-diagonal 2-D inv_mass: every
            # block inverted and Cholesky-factorised on its own with the reference's torch ops, then laid out as ONE
            # (D, D) operand pair for the full-mass kernels (thread-per-chain for D <= 16, tensor-core dense_lin above)
            blocks = [b.detach().to(torch.float32) for b in inv_mass]
            if any(b.dim() != 2 or b.shape[0] != b.shape[1] for b in blocks) or sum(b.shape[0] for b in blocks) != dim:
                raise RuntimeError('block-list inv_mass: square blocks whose sizes add up to %d' % dim)
            im = torch.block_diag(*blocks)
            tril = torch.block_diag(*[torch.linalg.cholesky(torch.inverse(b)) for b in blocks])
            s.kind = N.MASS_FULL
            self._keep['im'] = im.to(self.device).contiguous()
            self._keep['tril'] = tril.to(self.device).contiguous()
            s.inv_mass = self._keep['im'].data_ptr()
            s.mass_factor = self._keep['tril'].data_ptr()
        elif inv_mass.dim() == 1:
            if inv_mass.numel() != dim:
                raise RuntimeError('inv_mass must have %d entries' % dim)
            im = inv_mass.detach().to(torch.float32)
            sd = (1 / im) ** 0.5                       # mass = 1/inv_mass (:952); Normal(0, mass**0.5) (:201)
            s.kind = N.MASS_DIAG
            self._keep['im'] = im.to(self.device).contiguous()
            self._keep['sd'] = sd.to(self.device).contiguous()
            s.inv_mass = self._keep['im'].data_ptr()
            s.mass_factor = self._keep['sd'].data_ptr()
        elif inv_mass.dim() == 2:
            if tuple(inv_mass.shape) != (dim, dim):
                raise RuntimeError('inv_mass must be (%d, %d)' % (dim, dim))
            im = inv_mass.detach().to(torch.float32)
            mass = torch.inverse(im)                   # :950
            tril = torch.linalg.cholesky(mass)         # MultivariateNormal(0, mass).scale_tril (:199)
            s.kind = N.MASS_FULL
            self._keep['im'] = im.to(self.device).contiguous()
            self._keep['tril'] = tril.to(self.device).contiguous()
            s.inv_mass = self._keep['im'].data_ptr()
            s.mass_factor = self._keep['tril'].data_ptr()
        else:
            raise RuntimeError('inv_mass must be None, 1-D or 2-D')
        self.struct = s

    @property
    def kind(self):
        return self.struct.kind

    def ref(self):
        return C.byref(self.struct)


# A full (2-D) or block-list inv_mass costs a host inversion + Cholesky factorisation (samplers.py:942-952 does it once per
# sample() call).  Repeated calls with the SAME tensor object, unmodified (torch's version counter), reuse the device
# operands: the entry holds a reference to the caller's tensor(s), so a recycled address can never alias it.
_MASS_CACHE = []


def native_mass(inv_mass, dim, device):
    if isinstance(inv_mass, NativeMass):
        return inv_mass
    heavy = isinstance(inv_mass, list) or (torch.is_tensor(inv_mass) and inv_mass.dim() == 2)
    if not heavy:
        return NativeMass(inv_mass, dim, device)
    parts = inv_mass if isinstance(inv_mass, list) else [inv_mass]
    key = (tuple(id(t) for t in parts), tuple(t._version for t in parts), dim, str(torch.device(device)))
    for k, refs, nm in _MASS_CACHE:
        if k == key:
            return nm
    nm = NativeMass(inv_mass, dim, device)
    _MASS_CACHE.append((key, list(parts), nm))
    if len(_MASS_CACHE) > 4:
        _MASS_CACHE.pop(0)
    return nm


_SIDE_STREAMS = {}


def _side_stream(device):
    key = str(torch.device(device))
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def nuts_table(burn):
    """The five Python-double constants of samplers.py:659-671 for t = 1..burn+1 (gamma=.05, t0=10, kappa=.75)."""
    rows = []
    for n in range(burn + 1):
        t = n + 1
        w = (1 / (t + 10))
        rows.append([1 - w, w, (t ** 0.5) / 0.05, t ** -0.75, 1 - t ** -0.75])
    return torch.tensor(rows, dtype=torch.float64)


_NUTS_TABLES = {}


def nuts_table_device(burn, device):
    """The constants of nuts_table() on the device, built and uploaded once per (burn, device): the upload is a pageable
    host-to-device copy, i.e. a host synchronisation with everything queued on the stream -- per call it kept a sampler that
    is called in a loop from ever running ahead of the GPU."""
    key = (int(burn), str(torch.device(device)))
    t = _NUTS_TABLES.get(key)
    if t is None:
        if len(_NUTS_TABLES) > 16:
            _NUTS_TABLES.clear()
        t = _NUTS_TABLES[key] = nuts_table(burn).to(device)
    return t


def mass_windows(burn):
    """The slow windows of diagonal-mass adaptation over warm-up iterations 0 .. burn-1 as a list of (a, b) iteration ranges,
    with Stan's windowed-adaptation defaults: an initial buffer of 75 iterations, slow windows of 25 iterations doubling,
    a terminal buffer of 50.  A window is stretched to end at burn - 50 when the window after it (twice as long) would
    cross into the terminal buffer, i.e. end past burn - 50 (Stan's compute_next_window, whose inclusive last index
    makes its `>=` this `>`; the first window is never stretched).  When 75 + 25 + 50 > burn the buffers are
    int(0.15 * burn) and int(0.1 * burn) and the one window is what remains.  burn = 1000: [75, 100), [100, 150),
    [150, 250), [250, 450), [450, 950)."""
    burn = int(burn)
    if burn < 20:
        raise RuntimeError('adapt_mass needs burn >= 20 (got %d)' % burn)
    init, first, term = 75, 25, 50
    if init + first + term > burn:
        init, term = int(0.15 * burn), int(0.1 * burn)
        first = burn - init - term
    end = burn - term
    windows = []
    a, size = init, first
    b = a + size
    while True:
        windows.append((a, b))
        if b >= end:
            return windows
        a, size = b, 2 * size
        b = a + size
        if b + 2 * size > end:
            b = end


def nuts_table_restarted(burn):
    """nuts_table() with the dual averaging restarted at the end of every mass-adaptation window (mass_windows(burn)): the
    row of iteration n >= b, b the last window end <= n, holds the constants for t = n - b + 1."""
    ends = [b for _, b in mass_windows(burn)]
    rows, start = [], 0
    for n in range(burn + 1):
        if n in ends:
            start = n
        rows.append(n - start)                   # nuts_table()'s row n holds t = n + 1
    return nuts_table(burn)[rows]


def nuts_table_restarted_device(burn, device):
    """nuts_table_restarted() on the device, built and uploaded once per (burn, device) like nuts_table_device."""
    key = ('restarted', int(burn), str(torch.device(device)))
    t = _NUTS_TABLES.get(key)
    if t is None:
        if len(_NUTS_TABLES) > 16:
            _NUTS_TABLES.clear()
        t = _NUTS_TABLES[key] = nuts_table_restarted(burn).to(device)
    return t


def nuts_mu(step_size_init):
    """samplers.py:664 -- fp32 log of fp32(10*eps0), returned as a Python float."""
    return float(torch.log(10 * torch.FloatTensor([step_size_init])))


# ----------------------------------------------------------------------------------------------------------
# kernel entry points on torch tensors
# ----------------------------------------------------------------------------------------------------------
def _as_rows(x, ld, device):
    x = x.detach().to(device=device, dtype=torch.float32)
    if x.dim() == 1:
        x = x.unsqueeze(0)
    return N.pad_rows(x.contiguous(), ld)


def _eps_vector(step_size, C, device):
    if torch.is_tensor(step_size):
        e = step_size.detach().to(device=device, dtype=torch.float32).reshape(-1)
        if e.numel() == 1:
            e = e.expand(C)
        return e.contiguous().clone()
    return torch.full((C,), float(step_size), dtype=torch.float32, device=device)


def leapfrog(target, q, p, steps, step_size, inv_mass=None, return_trajectory=False, device=None):
    """Batched samplers.leapfrog (plain HMC branch).  q, p: (C, D) or (D,).  Returns (q_L, p_L) as (C, D), or
    the (L, C, D) trajectories when ``return_trajectory``."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    nm = native_mass(inv_mass, D, device)
    qd, pd = _as_rows(q, ld, device), _as_rows(p, ld, device)
    Cn = qd.shape[0]
    eps = _eps_vector(step_size, Cn, device)
    q_out, p_out = torch.empty_like(qd), torch.empty_like(pd)
    q_traj = p_traj = None
    if return_trajectory:
        q_traj = torch.empty((steps, Cn, ld), dtype=torch.float32, device=device)
        p_traj = torch.empty_like(q_traj)
    with torch.cuda.device(device):
        rc = lib.hmcx_leapfrog(nt.ref(), nm.ref(), N.ptr(qd), N.ptr(pd), N.ptr(eps), Cn, ld, int(steps),
                               N.ptr(q_out), N.ptr(p_out), N.ptr(q_traj), N.ptr(p_traj), N.stream_ptr(device))
    N.check(rc, 'hmcx_leapfrog')
    if return_trajectory:
        return q_traj[..., :D], p_traj[..., :D]
    return q_out[:, :D], p_out[:, :D]


def split_leapfrog(targets, q, p, steps, step_size, scheme, inv_mass=None, perms=None, seed=0, device=None):
    """Batched samplers.leapfrog with Integrator.SPLITTING / SPLITTING_RAND / SPLITTING_KMID (:494-603) on the list of
    data-split closures ``targets``.  q, p: (C, D) or (D,).  Returns the (L, C, D) trajectories of params and momentum
    (the state after every step).  SPLITTING_RAND: ``perms`` (C, M) injects the call's randperm(M) (:550), else Philox."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(targets, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    if isinstance(inv_mass, list) or (torch.is_tensor(inv_mass) and inv_mass.dim() != 1):
        raise NotImplementedError('split leapfrog: inv_mass None or 1-D')
    nm = native_mass(inv_mass, D, device)
    qd, pd = _as_rows(q, ld, device), _as_rows(p, ld, device)
    Cn, L = qd.shape[0], int(steps)
    eps = _eps_vector(step_size, Cn, device)
    rng = N.RngStruct()
    keep = []
    if perms is not None:
        pm = perms.detach().to(device=device, dtype=torch.int32).reshape(Cn, nt.num_splits).contiguous()
        rng.mode, rng.perms = N.RNG_INJECTED, pm.data_ptr()
        keep.append(pm)
    else:
        rng.mode, rng.seed = N.RNG_PHILOX, int(seed)
    q_traj = torch.zeros((L, Cn, ld), dtype=torch.float32, device=device)
    p_traj = torch.zeros_like(q_traj)
    with torch.cuda.device(device):
        rc = lib.hmcx_split_leapfrog(nt.ref(), nm.ref(), C.byref(rng), int(scheme), float(step_size), N.ptr(qd), N.ptr(pd),
                                     N.ptr(eps), Cn, ld, L, N.ptr(q_traj), N.ptr(p_traj), N.stream_ptr(device))
    N.check(rc, 'hmcx_split_leapfrog')
    torch.cuda.current_stream(device).synchronize()
    return q_traj[..., :D], p_traj[..., :D]


def hamiltonian(target, q, p, inv_mass=None, device=None):
    """Batched samplers.hamiltonian (sampler=HMC).  Returns (H (C,), nonfinite_flags (C,) uint8)."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    nm = native_mass(inv_mass, D, device)
    qd, pd = _as_rows(q, ld, device), _as_rows(p, ld, device)
    Cn = qd.shape[0]
    H = torch.empty(Cn, dtype=torch.float32, device=device)
    flags = torch.empty(Cn, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_hamiltonian(nt.ref(), nm.ref(), N.ptr(qd), N.ptr(pd), Cn, ld, N.ptr(H), N.ptr(flags),
                                  N.stream_ptr(device))
    N.check(rc, 'hmcx_hamiltonian')
    return H, flags


def gibbs(dim, num_chains, seed, iteration=0, inv_mass=None, chain_offset=0, device='cuda'):
    """Batched samplers.gibbs (sampler=HMC) from the in-kernel Philox stream."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device)
    ld = N.padded_ld(dim)
    nm = native_mass(inv_mass, dim, device)
    rng = N.RngStruct()
    rng.mode, rng.seed, rng.chain_offset = N.RNG_PHILOX, int(seed), int(chain_offset)
    p = torch.empty((num_chains, ld), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_gibbs(nm.ref(), C.byref(rng), dim, num_chains, ld, int(iteration), N.ptr(p),
                            N.stream_ptr(device))
    N.check(rc, 'hmcx_gibbs')
    return p[:, :dim]


class HMCResult:
    """Device-resident result of a batched run."""

    def __init__(self, samples, accepted, diverged, ham, step_size, num_rejected, dim, num_samples):
        self.samples_padded = samples            # (C, S-burn, ld)
        self.dim = dim
        self.accepted = accepted                 # (C, S) uint8
        self.diverged = diverged                 # (C, S) uint8
        self.ham = ham                           # (C, S, 2) or None
        self.step_size = step_size               # (C,) final per-chain eps
        self.num_rejected = num_rejected         # (C,) int32
        self.num_samples = num_samples

    @property
    def samples(self):
        if self.samples_padded is None:
            raise RuntimeError('this run kept no samples (keep_samples=False): use moment_sum / moment_sumsq')
        return self.samples_padded[..., :self.dim]

    @property
    def accept_rate(self):
        return 1.0 - self.num_rejected.double() / self.num_samples


def _run_device(params_init, device):
    """The device of an hmc_run / rmhmc_run call: ``device``, else params_init's CUDA device, else the current one.
    Refuses first when there is no CUDA device or no native library."""
    N.require_cuda()
    N.load_library()
    if device is None:
        device = params_init.device if params_init.is_cuda else torch.device('cuda', torch.cuda.current_device())
    return torch.device(device)


class _Run:
    """What one hmc_run / rmhmc_run call builds once and each of its launches reads: the device and its current stream,
    the native target, the (C, ld) rows of the initial and current state, the per-chain step sizes, the per-iteration
    outputs and ``keep_alive``, everything an asynchronous launch may still read when the call returns.  The caller then
    sets the sample block and the random-stream struct; hmc_run also the NUTS struct and its dual-averaging state, the
    integrator ``scheme``, ``tuning``, the element-wise workspace ``ws`` and ``num_folds``."""

    def __init__(self, nt, params_init, num_samples, num_steps_per_sample, step_size, burn, record_ham, device):
        self.lib = N.load_library()
        self.device, self.stream = device, N.stream_ptr(device)
        self.nt, self.D, self.ld = nt, nt.dim, N.padded_ld(nt.dim)
        self.S, self.L, self.burn = int(num_samples), int(num_steps_per_sample), int(burn)
        self.q_init = _as_rows(params_init, self.ld, device)
        self.Cn = Cn = self.q_init.shape[0]
        self.q_cur = self.q_init.clone()
        self.eps = _eps_vector(step_size, Cn, device)
        self.accepted = torch.empty((Cn, self.S), dtype=torch.uint8, device=device)
        self.diverged = torch.empty((Cn, self.S), dtype=torch.uint8, device=device)
        self.ham = torch.empty((Cn, self.S, 2), dtype=torch.float32, device=device) if record_ham else None
        self.num_rejected = torch.zeros(Cn, dtype=torch.int32, device=device)
        self.samples = self.rng = self.nuts = self.h_bar = self.eps_bar = self.scheme = self.ws = None
        self.tuning = self.num_folds = 0
        self.keep_alive = []

    def args(self, it0, it1):
        """The arguments every run entry takes from q_init to num_rejected, for iterations [it0, it1)."""
        return (N.ptr(self.q_init), N.ptr(self.q_cur), N.ptr(self.eps), self.Cn, self.ld, self.L, self.S, self.burn, it0,
                it1, N.ptr(self.samples), N.ptr(self.accepted), N.ptr(self.diverged), N.ptr(self.ham),
                N.ptr(self.num_rejected))


def _rng_struct(run, seed, chain_offset, normals, log_uniforms, perms=None, uniforms=None, jitter=False):
    """The random-stream struct of a run: Philox keyed by (seed, chain_offset + c, iteration), or -- when ``normals``
    (S, C, D) is given -- the injected stream: ``log_uniforms`` (S, C), SPLITTING_RAND's ``perms`` (S, C, M) if given and,
    for RMHMC with ``jitter``, the metric-jitter ``uniforms`` (S, C, J, D).  The device copies join run.keep_alive."""
    rng = N.RngStruct()
    if normals is None:
        rng.mode, rng.seed, rng.chain_offset = N.RNG_PHILOX, int(seed), int(chain_offset)
        return rng
    S, Cn, D, ld, device = run.S, run.Cn, run.D, run.ld, run.device
    z = normals.detach().to(device=device, dtype=torch.float32)
    if z.dim() == 2:
        z = z.unsqueeze(1)
    if tuple(z.shape) != (S, Cn, D):
        raise RuntimeError('normals must be (S, C, D) = (%d, %d, %d), got %s' % (S, Cn, D, tuple(z.shape)))
    z = N.pad_rows(z.contiguous(), ld)
    lu = log_uniforms.detach().to(device=device, dtype=torch.float32).reshape(S, Cn).contiguous()
    rng.mode, rng.normals, rng.log_uniforms = N.RNG_INJECTED, z.data_ptr(), lu.data_ptr()
    run.keep_alive += [z, lu]
    if perms is not None:
        if perms.dim() != 3 or tuple(perms.shape[:2]) != (S, Cn) or perms.shape[2] != run.nt.num_splits:
            raise RuntimeError('perms must be (S, C, M) = (%d, %d, %d), got %s'
                               % (S, Cn, run.nt.num_splits, tuple(perms.shape)))
        pm = perms.detach().to(device=device, dtype=torch.int32).contiguous()
        rng.perms = pm.data_ptr()
        run.keep_alive.append(pm)
    if jitter:
        if uniforms is None:
            raise RuntimeError('injected RMHMC with jitter needs the uniforms stream')
        u = uniforms.detach().to(device=device, dtype=torch.float32)
        if u.dim() == 3:
            u = u.unsqueeze(1)
        if u.dim() != 4 or tuple(u.shape[:2]) != (S, Cn) or u.shape[3] != D:
            raise RuntimeError('uniforms must be (S, C, J, D) = (%d, %d, J, %d), got %s' % (S, Cn, D, tuple(u.shape)))
        u = N.pad_rows(u.contiguous(), ld)
        rng.uniforms, rng.uniforms_per_iter = u.data_ptr(), u.shape[2]
        run.keep_alive.append(u)
    return rng


def hmc_run(target, params_init, num_samples, num_steps_per_sample, step_size, burn=0, inv_mass=None,
            nuts=False, desired_accept_rate=0.8, seed=0, chain_offset=0, normals=None, log_uniforms=None,
            record_ham=False, out=None, device=None, tuning=0, eps_schedule=None, record_eps=False, scheme=None,
            perms=None, thin=1, moments=False, keep_samples=True, host_samples=False, host_windows=0, adapt_mass=False,
            mass_pool=None, hyper=None, gammas=None, temper=None, folds=None, fits=None):
    """The reference's sample() loop for sampler in {HMC, HMC_NUTS} as one persistent kernel over C chains.

    params_init (C, D) | (D,).  Randomness: in-kernel Philox keyed by (seed, chain_offset+c, iteration), or -- when
    ``normals`` (S, C, D) and ``log_uniforms`` (S, C) are given -- the injected stream (parity mode).
    ``out``: optional pre-allocated (C, S-burn, ld) fp32 tensor for the samples: a device tensor, or a PINNED host
    tensor (the kernel then streams the retained rows straight into it, see ``host_samples``).
    Bayesian-NN targets (an MLPRegression or the list of split descriptors): ``scheme`` selects the integrator
    (N.SCHEME_PLAIN / SPLIT_SYM / SPLIT_RAND / SPLIT_KMID); ``perms`` (S, C, M) injects SPLITTING_RAND's randperm.
    NUTS only: ``eps_schedule`` (S, C) forces the step size of every iteration (parity tests replay the reference's
    schedule); ``record_eps`` returns the kernel's own adapted step sizes in ``result.eps_trace`` (C, S).
    Sample sink (include/hmcx.h hmcx_sink_t; element-wise targets and Bayesian-NN targets): ``thin`` keeps every
    thin-th post-burn state, ``moments`` accumulates per-chain running sum / sum of squares over every post-burn
    iteration with compensated (Neumaier) summation (``result.moment_sum``, ``result.moment_sumsq``: fp64 tensors
    relative error ~ n*eps^2 instead of the naive n*eps; ``result.moment_count``), ``keep_samples=False`` stores no
    samples at all, ``host_samples=True`` makes the kernel stream the retained rows straight into pinned host memory
    (the reference's ``store_on_GPU=False``, samplers.py:1008-1012) -- ``result.samples`` is then a CPU tensor, valid
    after a stream synchronisation.
    ``adapt_mass`` (NUTS, sink-capable target, inv_mass None or 1-D): adapt one diagonal inv_mass shared by all chains
    during warm-up (DESIGN §3.13).  Each window of mass_windows(burn) is a sink launch accumulating the chains' moments,
    followed by hmcx_adapt_diag_mass, which pools them into the mass the next launch reads and restarts the dual averaging;
    the last launch runs the rest of the warm-up and the sampling phase with the sink options above.  All on the current
    stream, no host synchronisation.  ``result.inv_mass`` (D,), ``result.inv_mass_trace`` (K, D), ``result.mass_windows``.
    ``mass_pool``: callable mapping each (C_local, ld) window sum to the (C, ld) sum of all chains in global order
    (distributed.sample_chains_sharded passes an all-gather), so that every rank pools every chain into the same mass.
    ``hyper`` (Bayesian-NN targets with a ``scheme``): Gamma hyperpriors on the precisions, a list of 2L + 1 entries --
    the parameter tensors in tau_list order, then tau_out -- each None (fixed) or (a, b) (shape, rate), Gibbs-updated
    inside the kernel after every MH step (include/hmcx.h hmcx_hyper_t, DESIGN §3.15).  Injected mode takes ``gammas``
    (S, C, 2L + 1) fp64 standard-gamma draws.  The result gains ``tau_list_trace`` (C, keep, 2L), ``tau_out_trace``
    (C, keep) -- on the device whatever ``host_samples`` says -- the final state ``tau_list_final`` (C, 2L),
    ``tau_out_final`` (C,), and ``hyper`` (the list as given, which ``sensitivity.log_components`` reads).
    ``temper`` (Bayesian-NN targets with a ``scheme``): replica exchange, a dict with ``betas`` (T Python floats, 1.0 first,
    strictly decreasing), ``swap_every`` and ``swap_log_uniforms`` ((rounds, R, T - 1) fp64 or None: Philox).  The C = R T
    rows are R ladders, row r T + t at beta_t (include/hmcx.h hmcx_temper_t, DESIGN §3.17): the run goes in windows of
    ``swap_every`` iterations with a swap round (hmcx_temper_swap) after each window but the last.  ``samples`` / ``out``
    hold the beta = 1 rows only, (R, keep, ld); the result gains ``betas``, ``swap_accepted`` (rounds, R, T - 1) int8,
    ``swap_ll`` (rounds, C) fp64 and ``swap_rate`` (T - 1,).
    ``folds`` (an MLPTarget with ``scheme`` PLAIN): K-fold refits, an (N,) integer tensor assigning each data row to a fold
    0 .. K-1 or to -1 (never left out).  The target becomes ``fold_targets(target, folds)`` and one hmcx_split_run_folds
    launch runs chain g = chain_offset + c on fold g mod K's training rows (DESIGN §3.18).  The result gains ``folds``
    (the assignment, on the device) and ``num_folds``.
    ``fits`` (instead of ``target`` and ``folds``): the list of K MLPTargets of the fits themselves, sharing the network,
    prior and settings -- the fold path with the training sets given directly (sbc.fit passes K copies of one target, each
    holding its own simulated y).  Chain g = chain_offset + c samples fits[g mod K].
    """
    device = _run_device(params_init, device)
    num_folds = 0
    if folds is not None or fits is not None:
        if scheme != N.SCHEME_PLAIN or temper is not None or hyper is not None or adapt_mass:
            raise NotImplementedError('K-fold runs: the plain integrator on an MLPTarget, without replica exchange, '
                                      'hyperpriors or adapt_mass')
        if folds is not None:
            folds = torch.as_tensor(folds).to(device=device, dtype=torch.int64)
            fits = fold_targets(target, folds.cpu())
        target = fits
        num_folds = len(fits)
    nt = native_target(target, device)
    nm = native_mass(inv_mass, nt.dim, device)
    run = _Run(nt, params_init, num_samples, num_steps_per_sample, step_size, burn, record_ham, device)
    D, ld, Cn, S, burn = run.D, run.ld, run.Cn, run.S, run.burn
    if run.q_init.shape[1] != ld or params_init.shape[-1] != D:
        raise RuntimeError('params_init last dimension must be %d' % D)
    thin = int(thin)
    if thin < 1:
        raise RuntimeError('thin must be >= 1')
    host_out = None
    if out is not None and not out.is_cuda:
        if not out.is_pinned():
            raise RuntimeError('a host `out` buffer must be pinned (page-locked) memory')
        if (int(host_windows) >= 2 and thin == 1 and not moments and keep_samples and scheme is None and ld <= 4096 and
                nt.struct.kind in (T.GaussianIso.kind, T.GaussianDiag.kind) and nm.kind != N.MASS_FULL and normals is None):
            # windowed delivery: the run is cut into `host_windows` windows of iterations; each window's sample slots
            # leave for the pinned block through the COPY ENGINE on a second stream while the next window computes
            # (hmcx_copy_rows_async).  Costs a device staging block of the samples' size; delivers at the DMA rate
            host_out, out = out, None
        else:
            host_samples = True                    # caller-provided pinned sample block: the kernel streams into it
    if adapt_mass:
        if not nuts:
            raise RuntimeError('adapt_mass re-tunes the step size after each mass update: it needs NUTS (dual averaging)')
        if nm.kind == N.MASS_FULL or host_out is not None:
            raise NotImplementedError('adapt_mass: inv_mass None or 1-D, no windowed copy-engine delivery')
    use_sink = thin > 1 or moments or not keep_samples or host_samples
    keep = 1 + (S - burn - 1) // thin
    if temper is not None:
        if scheme is None or hyper is not None or adapt_mass:
            raise NotImplementedError('replica exchange: Bayesian-NN targets, without hyperpriors or adapt_mass')
        if Cn % len(temper['betas']) != 0:
            raise ValueError('replica exchange: C = %d rows is not a multiple of T = %d' % (Cn, len(temper['betas'])))
    Cs = Cn if temper is None else Cn // len(temper['betas'])      # rows of the sample block
    if not keep_samples:
        samples = None
    elif host_samples and out is None:
        # pinned host memory is device-addressable under unified virtual addressing: the kernel's st.global.cs rows go
        # over PCIe while the chains keep running (no device-side sample buffer, no separate D2H copy)
        samples = torch.empty((Cs, keep, ld), dtype=torch.float32, pin_memory=True)
    elif out is None:
        samples = torch.empty((Cs, keep, ld), dtype=torch.float32, device=device)
    else:
        samples = out
        if tuple(samples.shape) != (Cs, keep, ld) or samples.dtype != torch.float32 or not samples.is_contiguous():
            raise RuntimeError('out must be a contiguous fp32 (%s, S-burn, ld) tensor' % ('C' if temper is None else 'R'))
    run.samples = samples
    run.rng = _rng_struct(run, seed, chain_offset, normals, log_uniforms, perms=perms)

    nuts_s = run.nuts = N.NutsStruct()
    eps_trace = None
    if not torch.is_tensor(step_size):
        nuts_s.step_size_init = float(step_size)           # the double the reference divides in its split drifts
    if nuts:
        table = nuts_table_restarted_device(burn, device) if adapt_mass else nuts_table_device(burn, device)
        run.h_bar = torch.zeros(Cn, dtype=torch.float64, device=device)
        run.eps_bar = torch.ones(Cn, dtype=torch.float64, device=device)
        nuts_s.enabled = 1
        nuts_s.desired_accept_rate = float(desired_accept_rate)
        nuts_s.mu = nuts_mu(step_size if not torch.is_tensor(step_size) else float(step_size.reshape(-1)[0]))
        nuts_s.table, nuts_s.h_bar, nuts_s.eps_bar = table.data_ptr(), run.h_bar.data_ptr(), run.eps_bar.data_ptr()
        run.keep_alive += [table, run.h_bar, run.eps_bar]
        if eps_schedule is not None:
            sched = eps_schedule.detach().to(device=device, dtype=torch.float32).reshape(S, Cn).contiguous()
            nuts_s.eps_schedule = sched.data_ptr()
            run.keep_alive.append(sched)
        if record_eps:
            eps_trace = torch.zeros((Cn, S), dtype=torch.float32, device=device)
            nuts_s.eps_trace = eps_trace.data_ptr()

    msum = msq = msum_lo = msq_lo = None
    sink = None
    if use_sink:
        sink = N.SinkStruct()
        sink.thin = thin
        if moments:
            msum, msq, msum_lo, msq_lo = (torch.zeros((Cn, ld), dtype=torch.float32, device=device) for _ in range(4))
            sink.sum, sink.sumsq = msum.data_ptr(), msq.data_ptr()
            sink.sum_lo, sink.sumsq_lo = msum_lo.data_ptr(), msq_lo.data_ptr()
    hyper_s = None
    if hyper is not None:
        if scheme is None:
            raise NotImplementedError('hyperpriors: Bayesian-NN targets only')
        desc = nt.mlp_desc
        K = 2 * desc.num_layers
        if len(hyper) != K + 1:
            raise RuntimeError('hyper needs %d entries (the parameter tensors, then tau_out)' % (K + 1))
        hyper_s = N.HyperStruct()
        for k, ab in enumerate(hyper):
            if ab is not None:
                hyper_s.sampled[k] = 1
                hyper_s.a[k], hyper_s.b[k] = float(ab[0]), float(ab[1])
        tau = torch.tensor([float(t) for t in desc.tau_list], dtype=torch.float32).to(device).repeat(Cn, 1).contiguous()
        tau_out = torch.full((Cn,), desc.tau_out, dtype=torch.float32, device=device)
        tau_trace = torch.zeros((Cn, keep, K), dtype=torch.float32, device=device)
        tau_out_trace = torch.zeros((Cn, keep), dtype=torch.float32, device=device)
        hyper_s.tau, hyper_s.tau_out = tau.data_ptr(), tau_out.data_ptr()
        hyper_s.tau_trace, hyper_s.tau_out_trace = tau_trace.data_ptr(), tau_out_trace.data_ptr()
        run.keep_alive += [tau, tau_out, tau_trace, tau_out_trace]
        if run.rng.mode == N.RNG_INJECTED:
            if gammas is None or tuple(gammas.shape) != (S, Cn, K + 1):
                raise RuntimeError('injected hyperpriors need gammas (S, C, 2L + 1) = (%d, %d, %d)' % (S, Cn, K + 1))
            gm = gammas.detach().to(device=device, dtype=torch.float64).contiguous()
            hyper_s.gammas = gm.data_ptr()
            run.keep_alive.append(gm)
    run.scheme, run.tuning, run.num_folds = scheme, int(tuning), num_folds
    mass_out = None
    temper_out = None
    with torch.cuda.device(device):
        if scheme is None:
            ws_bytes = run.lib.hmcx_hmc_workspace_bytes(nt.ref(), nm.ref(), Cn, ld)
            run.ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=device) if ws_bytes else None
        if temper is not None:
            temper_out = _tempered_launches(run, nm, sink, temper)
        elif adapt_mass:
            if sink is None:
                sink = N.SinkStruct()
                sink.thin = 1
            mass_out = _adapted_launches(run, nm, sink, hyper_s, mass_pool)
        elif host_out is not None and sink is None:
            if tuple(host_out.shape) != (Cn, keep, ld) or host_out.dtype != torch.float32 or not host_out.is_contiguous():
                raise RuntimeError('out must be a contiguous fp32 (C, S-burn, ld) tensor')
            W = min(int(host_windows), S)
            main = torch.cuda.current_stream(device)
            side = _side_stream(device)
            pitch, slot_bytes = keep * ld * 4, ld * 4
            for w in range(W):
                a, b = (S * w) // W, (S * (w + 1)) // W
                _launch(run, a, b, nm.ref(), None)
                lo = 0 if a == 0 else max(a - burn, 1)               # slots this window wrote: 0 = params_init (:959),
                hi = max(b - burn, 1 if a == 0 else lo)              # n - burn for every iteration n > burn
                if hi > lo:
                    ev = torch.cuda.Event()
                    ev.record(main)
                    side.wait_event(ev)
                    rc = run.lib.hmcx_copy_rows_async(C.c_void_p(host_out.data_ptr() + lo * slot_bytes), pitch,
                                                      C.c_void_p(samples.data_ptr() + lo * slot_bytes), pitch,
                                                      (hi - lo) * slot_bytes, Cn, C.c_void_p(side.cuda_stream))
                    N.check(rc, 'hmcx_copy_rows_async')
            done = torch.cuda.Event()
            done.record(side)
            main.wait_event(done)                       # the caller's stream sees the delivered block
            run.keep_alive.append(samples)
            samples = host_out
        else:
            _launch(run, 0, S, nm.ref(), sink, hyper_s)
    res = HMCResult(samples, run.accepted, run.diverged, run.ham, run.eps, run.num_rejected, D, S)
    res.eps_trace = eps_trace
    res.thin = thin
    # compensated running sums: hi + lo combined in fp64 (relative error ~2^-46 whatever the run length)
    res.moment_sum = None if msum is None else (msum.double() + msum_lo.double())[:, :D]
    res.moment_sumsq = None if msq is None else (msq.double() + msq_lo.double())[:, :D]
    res.moment_count = S - burn - 1
    res.final_state = run.q_cur[:, :D]
    if nuts:
        res.eps_bar, res.h_bar = run.eps_bar, run.h_bar
    if mass_out is not None:
        res.inv_mass_trace, res.mass_windows = mass_out
        res.inv_mass = res.inv_mass_trace[-1]
    if hyper_s is not None:
        res.tau_list_trace, res.tau_out_trace = tau_trace, tau_out_trace
        res.tau_list_final, res.tau_out_final = tau, tau_out
        res.hyper = list(hyper)
    if folds is not None:
        res.folds, res.num_folds = folds, num_folds
    if temper_out is not None:
        res.betas, res.swap_accepted, res.swap_ll = temper_out
        a = res.swap_accepted
        tried = (a >= 0).sum(dim=(0, 1))
        res.swap_rate = (a == 1).sum(dim=(0, 1)).double() / tried.clamp_min(1).double()
    res._keep_alive = run.keep_alive      # buffers the asynchronous kernel still reads
    return res


def swap_rounds(num_samples, swap_every):
    """The number of swap rounds of a tempered run: one after every window of ``swap_every`` iterations but the last."""
    return max(0, -(-int(num_samples) // int(swap_every)) - 1)


def _tempered_launches(run, nm, sink, temper):
    """hmc_run with replica exchange: the windows [k E, min(S, (k + 1) E)) of E = swap_every iterations, each a tempered
    sink launch (hmcx_split_run_temper) that leaves the untempered log-likelihood of every row in swap_ll[k], followed by
    swap round k (hmcx_temper_swap) when iterations remain.  All on the current stream, no host synchronisation.  Returns
    (betas (T,) fp64, swap_accepted (rounds, R, T - 1) int8, swap_ll (rounds, C) fp64)."""
    betas = [float(b) for b in temper['betas']]
    T, E = len(betas), int(temper['swap_every'])
    R, rounds = run.Cn // T, swap_rounds(run.S, E)
    tau0 = run.nt.mlp_desc.tau_out
    ts = N.TemperStruct()
    ts.num_temps = T
    for t, b in enumerate(betas):
        ts.tau_out[t] = b * tau0                 # the Python-double product, rounded to fp32 as MLPTarget(tau_out=b*tau0)
    sink_s = sink
    if sink_s is None:
        sink_s = N.SinkStruct()
        sink_s.thin = 1
    swap_acc = torch.empty((rounds, R, T - 1), dtype=torch.int8, device=run.device)
    swap_ll = torch.empty((rounds, run.Cn), dtype=torch.float64, device=run.device)
    lu = temper.get('swap_log_uniforms')
    if lu is not None:
        if tuple(lu.shape) != (rounds, R, T - 1):
            raise ValueError('swap_log_uniforms must be (rounds, R, T - 1) = (%d, %d, %d), got %s'
                             % (rounds, R, T - 1, tuple(lu.shape)))
        lu = lu.detach().to(device=run.device, dtype=torch.float64).contiguous()
    srng = N.RngStruct()
    srng.mode = N.RNG_INJECTED if lu is not None else N.RNG_PHILOX
    srng.seed, srng.chain_offset = run.rng.seed, run.rng.chain_offset
    cb = (C.c_double * T)(*betas)
    run.keep_alive += [swap_acc, swap_ll, lu, ts, sink_s, srng, cb]
    for k in range(rounds + 1):
        ts.ll_out = swap_ll[k].data_ptr() if k < rounds else None
        _launch(run, k * E, min(run.S, (k + 1) * E), nm.ref(), sink_s, temper=ts)
        if k < rounds and T > 1:
            rc = run.lib.hmcx_temper_swap(N.ptr(run.q_cur), run.Cn, run.ld, T, cb, N.ptr(swap_ll[k]), k, C.byref(srng),
                                          None if lu is None else C.c_void_p(lu[k].data_ptr()), N.ptr(swap_acc[k]),
                                          run.stream)
            N.check(rc, 'hmcx_temper_swap')
    return torch.tensor(betas, dtype=torch.float64), swap_acc, swap_ll


def _window_hyper(hyper_s, it0, Cn, groups):
    """The hyperprior struct of a launch starting at iteration it0: the injected gamma draws (rows of Cn * groups fp64)
    move to row it0."""
    if hyper_s is None or not hyper_s.gammas or it0 == 0:
        return hyper_s
    h = N.HyperStruct.from_buffer_copy(hyper_s)
    h.gammas = hyper_s.gammas + it0 * Cn * groups * 8
    return h


def _window_rng(rng, it0, Cn, ld, num_splits):
    """The random-stream struct of a launch starting at iteration it0: injected streams are indexed from the launch's first
    iteration, so their pointers move to row it0."""
    if rng.mode != N.RNG_INJECTED or it0 == 0:
        return rng
    r = N.RngStruct.from_buffer_copy(rng)
    r.normals = rng.normals + it0 * Cn * ld * 4
    r.log_uniforms = rng.log_uniforms + it0 * Cn * 4
    if rng.perms:
        r.perms = rng.perms + it0 * Cn * num_splits * 4
    return r


def _launch(run, it0, it1, mass_ref, sink, hyper=None, temper=None):
    """Iterations [it0, it1) of ``run`` as one launch on the run's stream: the only call of a libhmcx run entry.  The
    injected streams (and injected gamma draws) move to row it0; the per-launch struct copies join run.keep_alive.
    Descriptor targets (``run.scheme`` None): hmcx_hmc_run_sink, ``sink`` None for a plain run.
    Bayesian-NN targets: hmcx_split_run_folds for K-fold runs, hmcx_split_run_temper with ``temper``, else
    hmcx_split_run_hyper (``sink`` and ``hyper`` may be None)."""
    rng = _window_rng(run.rng, it0, run.Cn, run.ld, run.nt.num_splits)
    h = None if hyper is None else _window_hyper(hyper, it0, run.Cn, 2 * run.nt.mlp_desc.num_layers + 1)
    run.keep_alive += [rng, h]
    head = (run.nt.ref(), mass_ref, C.byref(rng), C.byref(run.nuts))
    sink = None if sink is None else C.byref(sink)
    lib = run.lib
    if run.scheme is None:
        name = 'hmcx_hmc_run_sink'
        rc = lib.hmcx_hmc_run_sink(*head, *run.args(it0, it1), run.tuning, N.ptr(run.ws), sink, run.stream)
    elif run.num_folds:
        name = 'hmcx_split_run_folds'
        rc = lib.hmcx_split_run_folds(*head, int(run.scheme), *run.args(it0, it1), sink, run.num_folds, run.stream)
    elif temper is not None:
        name = 'hmcx_split_run_temper'
        rc = lib.hmcx_split_run_temper(*head, int(run.scheme), *run.args(it0, it1), sink, C.byref(temper), run.stream)
    else:
        name = 'hmcx_split_run_hyper'
        rc = lib.hmcx_split_run_hyper(*head, int(run.scheme), *run.args(it0, it1), sink, None if h is None else C.byref(h),
                                      run.stream)
    N.check(rc, name)


def _adapted_launches(run, nm, sink, hyper_s, mass_pool):
    """hmc_run with adapt_mass: [0, a_1) and every window [a_k, b_k) of mass_windows(burn), each window followed by
    hmcx_adapt_diag_mass, then [b_K, S) with the caller's sink (and the hyperprior state ``hyper_s``, if any).  Every launch is a sink launch (mu_chain and moments_all
    are read by the sink forms only); the launches chain through q_cur, eps, the dual-averaging state and, for element-wise
    targets, the log p workspace.  Returns (inv_mass_trace (K, D), windows)."""
    windows = mass_windows(run.burn)
    K = len(windows)
    Cn, ld, device = run.Cn, run.ld, run.device
    trace = torch.zeros((K, ld), dtype=torch.float32, device=device)          # row k: inv_mass after window k
    factor = torch.zeros((K, ld), dtype=torch.float32, device=device)         # row k: its sqrt(1 / inv_mass)
    acc = [torch.zeros((Cn, ld), dtype=torch.float32, device=device) for _ in range(4)]
    mu_chain = torch.zeros(Cn, dtype=torch.float64, device=device)
    wsink = N.SinkStruct()
    wsink.thin = sink.thin
    wsink.sum, wsink.sumsq, wsink.sum_lo, wsink.sumsq_lo = (t.data_ptr() for t in acc)
    wsink.moments_all = 1
    masses = []
    for k in range(K):
        m = N.MassStruct()
        m.kind, m.inv_mass, m.mass_factor = N.MASS_DIAG, trace[k].data_ptr(), factor[k].data_ptr()
        masses.append(m)
    run.keep_alive += [trace, factor, mu_chain, wsink, masses] + acc
    if run.scheme is None:
        run.keep_alive.append(run.ws)

    def launch(it0, it1, mass_ref, sink_s, per_chain_mu):
        run.nuts.mu_chain = mu_chain.data_ptr() if per_chain_mu else None
        _launch(run, it0, it1, mass_ref, sink_s, hyper_s)

    mass_ref = nm.ref()
    launch(0, windows[0][0], mass_ref, sink, False)
    for k, (a, b) in enumerate(windows):
        launch(a, b, mass_ref, wsink, k > 0)
        sums = acc if mass_pool is None else [mass_pool(t).contiguous() for t in acc]
        if mass_pool is not None:
            run.keep_alive.extend(sums)
        rc = run.lib.hmcx_adapt_diag_mass(*(N.ptr(t) for t in sums), sums[0].shape[0], ld, run.D, b - a, N.ptr(run.eps),
                                          Cn, N.ptr(trace[k]), N.ptr(factor[k]), N.ptr(mu_chain), N.ptr(run.h_bar),
                                          N.ptr(run.eps_bar), run.stream)
        N.check(rc, 'hmcx_adapt_diag_mass')
        if mass_pool is not None:                  # the kernel zeroed the gathered copies; the next window starts from zero
            for t in acc:
                t.zero_()
        mass_ref = C.byref(masses[k])
    launch(windows[-1][1], run.S, mass_ref, sink, True)
    return trace[:, :run.D], windows


def hyper_gamma_draws(seed, num_chains, iter_begin, iter_end, shapes, chain_offset=0, device='cuda'):
    """The Philox-mode standard-gamma draws of the hyperprior kernels (hmcx_hyper_gamma_draws): (iter_end - iter_begin,
    num_chains, K) fp64, entry [n, c, k] the Gamma(shapes[k], 1) draw of group k for chain chain_offset + c at
    iteration iter_begin + n."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device)
    K = len(shapes)
    sh = (C.c_double * max(K, 1))(*[float(v) for v in shapes])
    out = torch.empty((int(iter_end) - int(iter_begin), int(num_chains), K), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_hyper_gamma_draws(int(seed), int(chain_offset), int(num_chains), int(iter_begin), int(iter_end), K,
                                        sh, N.ptr(out), N.stream_ptr(device))
    N.check(rc, 'hmcx_hyper_gamma_draws')
    return out


def grad_log_prob(target, q, split=-1, want_grad=True, want_log_prob=True, device=None):
    """Batched collect_gradients (samplers.py:33-66): (grad (C, D), log_prob (C,)) of C parameter vectors for a
    Bayesian-NN target; ``split`` selects one data split (-1: the whole potential)."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    qd = _as_rows(q, ld, device)
    Cn = qd.shape[0]
    g = torch.empty_like(qd) if want_grad else None
    lp = torch.empty(Cn, dtype=torch.float32, device=device) if want_log_prob else None
    with torch.cuda.device(device):
        rc = lib.hmcx_grad_log_prob(nt.ref(), N.ptr(qd), Cn, ld, int(split), N.ptr(g), N.ptr(lp), N.stream_ptr(device))
    N.check(rc, 'hmcx_grad_log_prob')
    return (g[:, :D] if want_grad else None), lp


def mlp_predict(target, samples, device=None):
    """Batched predict_model (samplers.py:1468-1562): samples (S, D) -> (pred (S, N, O), log_prob (S,))."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (samples.device if samples.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    sd = _as_rows(samples, ld, device)
    S = sd.shape[0]
    m = nt.mlp_struct
    pred = torch.empty((S, m.num_rows, m.widths[m.num_layers]), dtype=torch.float32, device=device)   # logits / log-probs
    lp = torch.empty(S, dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_mlp_predict(nt.ref(), N.ptr(sd), S, ld, N.ptr(pred), N.ptr(lp), N.stream_ptr(device))
    N.check(rc, 'hmcx_mlp_predict')
    return pred, lp


def const_metric(target, softabs, softabs_const):
    """The metric of a Gaussian target without jitter is one matrix: evaluate it ONCE on the host with the reference's
    own torch ops (fisher, samplers.py:108-121: autograd Hessian of the descriptor, eigh + coth map for SOFTABS) and
    derive what the kernels consume: G^-1 (the metric solve of cholesky_inverse :146-148 as a matrix), chol(G) (gibbs
    :183-184 through MultivariateNormal's scale_tril) and log det G (:726 / :728)."""
    D = target.dim
    # -Hessian of the quadratic log-density; what torch.autograd.functional.hessian(target, q) (:108) returns at ANY q
    # (tests/test_targets.py::test_const_metric_matches_the_oracle_fisher) without its D backward passes
    if isinstance(target, T.GaussianFull):
        fish = target.prec.detach().clone()
    elif isinstance(target, T.GaussianDiag):
        fish = torch.diag(target.inv_var.detach().to(torch.float32))
    elif isinstance(target, T.GaussianIso):
        fish = torch.eye(D, dtype=torch.float32)
    else:
        fish = -torch.autograd.functional.hessian(target, torch.zeros(D), create_graph=False)
    if softabs:
        lam, vec = torch.linalg.eigh(fish, UPLO='L')
        abs_lam = (1. / torch.tanh(softabs_const * lam)) * lam
        fish = torch.matmul(vec, torch.matmul(abs_lam.diag(), vec.t()))
        log_det = float(abs_lam.log().sum())
    else:
        log_det = float(torch.slogdet(fish)[1])
    lower = torch.linalg.cholesky(fish)
    ginv = torch.cholesky_inverse(lower.double()).float()        # (L L^T)^-1 from the reference's fp32 factor
    return ginv.contiguous(), lower.contiguous(), log_det


# The constant metric costs an eigh / Cholesky / inverse on the host (the reference pays them at EVERY fisher() call).  Repeated
# runs on the SAME target object, unmodified, reuse the device operands -- keyed like _MASS_CACHE; the entry holds the target.
_METRIC_CACHE = []


def const_metric_device(target, softabs, softabs_const, device):
    tensors = [t for t in (getattr(target, 'prec', None), getattr(target, 'inv_var', None)) if torch.is_tensor(t)]
    key = (id(target), tuple(id(t) for t in tensors), tuple(t._version for t in tensors), bool(softabs),
           float(softabs_const) if softabs else None, str(torch.device(device)))
    for k, _, val in _METRIC_CACHE:
        if k == key:
            return val
    ginv, lower, log_det = const_metric(target, softabs, softabs_const)
    val = (ginv.to(device), lower.to(device), log_det)
    _METRIC_CACHE.append((key, target, val))
    if len(_METRIC_CACHE) > 4:
        _METRIC_CACHE.pop(0)
    return val


def _rmhmc_is_dense(target, jitter, jacdiag=False):
    """Gaussian targets without jitter have a constant metric: the tensor-core path (GaussianFull at any D; GaussianIso /
    GaussianDiag above D = 16, below they stay on the thread-per-chain kernel).  Everything else -- Funnel, jitter,
    Metric.JACOBIAN_DIAG (depends on the gradient, i.e. on the position) -- assembles and factorises its metric inside
    the kernel: hmcx_rmhmc_run (D <= 16 one thread per chain, D <= 64 one CTA per chain)."""
    if jitter is not None or jacdiag or os.environ.get('HMCX_RMHMC_FORCE_CTA') == '1':
        return False
    if isinstance(target, T.GaussianFull):
        return True
    return isinstance(target, (T.GaussianIso, T.GaussianDiag)) and target.dim > 16


def rmhmc_run(target, params_init, num_samples, num_steps_per_sample, step_size, burn=0, jitter=None,
              softabs_const=None, explicit_binding_const=100, fixed_point_threshold=1e-5,
              fixed_point_max_iterations=1000, jitter_max_tries=10, explicit=True, softabs=False, jacdiag=False, seed=0,
              chain_offset=0, normals=None, log_uniforms=None, uniforms=None, record_ham=False, device=None):
    """The reference's sample() loop for sampler=RMHMC over C chains (one thread per chain).

    Injected (parity) mode: ``normals`` (S, C, D), ``log_uniforms`` (S, C) and -- when ``jitter`` is not None --
    ``uniforms`` (S, C, J, D): the ``torch.rand(D)`` jitter draws of every ``fisher`` call of iteration n in the
    reference's order (J = 8*L+3 for the explicit integrator)."""
    device = _run_device(params_init, device)
    nt = native_target(target, device)
    if explicit and torch.is_tensor(step_size) and step_size.numel() > 1:
        s = step_size.detach().reshape(-1)
        if not bool((s == s[0]).all()):
            # every kernel applies ONE binding rotation c, s = cos/sin(2 * omega * step_size) (:435-436) to all chains
            raise NotImplementedError('the explicit RMHMC integrator takes one step size for all chains')
    run = _Run(nt, params_init, num_samples, num_steps_per_sample, step_size, burn, record_ham, device)
    D, ld, Cn, S, burn = run.D, run.ld, run.Cn, run.S, run.burn
    run.samples = torch.empty((Cn, S - burn, ld), dtype=torch.float32, device=device)
    if softabs and softabs_const is None:
        raise RuntimeError('Metric.SOFTABS needs softabs_const')

    cfg = _rmhmc_cfg(D, step_size, jitter, softabs_const, explicit_binding_const, fixed_point_threshold,
                     fixed_point_max_iterations, jitter_max_tries, explicit, softabs, jacdiag)
    rng = run.rng = _rng_struct(run, seed, chain_offset, normals, log_uniforms, uniforms=uniforms,
                                jitter=jitter is not None)
    with torch.cuda.device(device):
        if _rmhmc_is_dense(nt.target, jitter, jacdiag):
            ginv_d, lower_d, log_det = const_metric_device(nt.target, softabs, softabs_const, device)
            gm = N.ConstMetricStruct()
            gm.metric_inv, gm.metric_chol, gm.log_det = ginv_d.data_ptr(), lower_d.data_ptr(), log_det
            ws = torch.empty(run.lib.hmcx_rmhmc_dense_workspace_bytes(Cn, D) // 4, dtype=torch.float32, device=device)
            run.keep_alive += [ginv_d, lower_d, ws]
            rc = run.lib.hmcx_rmhmc_dense_run(nt.ref(), C.byref(cfg), C.byref(gm), C.byref(rng), *run.args(0, S),
                                              N.ptr(ws), run.stream)
            N.check(rc, 'hmcx_rmhmc_dense_run')
        else:
            rc = run.lib.hmcx_rmhmc_run(nt.ref(), C.byref(cfg), C.byref(rng), *run.args(0, S), run.stream)
            N.check(rc, 'hmcx_rmhmc_run')
    res = HMCResult(run.samples, run.accepted, run.diverged, run.ham, run.eps, run.num_rejected, D, S)
    res.eps_trace = None
    res.final_state = run.q_cur[:, :D]
    res._keep_alive = run.keep_alive
    return res


def _rmhmc_cfg(D, step_size, jitter, softabs_const, explicit_binding_const, fixed_point_threshold,
               fixed_point_max_iterations, jitter_max_tries, explicit, softabs, jacdiag):
    cfg = N.RmhmcStruct()
    cfg.integrator = 1 if explicit else 2
    cfg.metric = 3 if jacdiag else (2 if softabs else 1)
    cfg.softabs_const = float(softabs_const) if softabs_const is not None else 0.0
    cfg.jitter = float(jitter) if jitter is not None else -1.0
    cfg.pi_term = float(D * torch.log(2. * torch.tensor(math.pi)))                              # samplers.py:711-712
    eps0 = float(step_size) if not torch.is_tensor(step_size) else float(step_size.reshape(-1)[0])
    cfg.cos_2we = float(torch.cos(torch.FloatTensor([2 * explicit_binding_const * eps0])))    # :435
    cfg.sin_2we = float(torch.sin(torch.FloatTensor([2 * explicit_binding_const * eps0])))    # :436
    cfg.fixed_point_threshold = float(fixed_point_threshold)
    cfg.fixed_point_max_iterations = int(fixed_point_max_iterations)
    cfg.jitter_max_tries = int(jitter_max_tries)
    return cfg


def _standalone_rng(jitter, uniforms, seed, Cn, D, ld, device, keep):
    """Jitter draws of a stand-alone RMHMC call: injected ``uniforms`` (C, J, D) / (J, D) in fisher() call order, else
    Philox keyed by ``seed``."""
    rng = N.RngStruct()
    if jitter is not None and uniforms is not None:
        u = uniforms.detach().to(device=device, dtype=torch.float32)
        if u.dim() == 2:
            u = u.unsqueeze(0)
        if u.dim() != 3 or u.shape[0] != Cn or u.shape[2] != D:
            raise RuntimeError('uniforms must be (C, J, D) = (%d, J, %d), got %s' % (Cn, D, tuple(u.shape)))
        u = N.pad_rows(u.contiguous(), ld)
        rng.mode, rng.uniforms, rng.uniforms_per_iter = N.RNG_INJECTED, u.data_ptr(), u.shape[1]
        keep.append(u)
    else:
        rng.mode, rng.seed = N.RNG_PHILOX, int(seed)
    return rng


def rmhmc_leapfrog(target, q, p, steps, step_size, jitter=None, softabs_const=None, explicit_binding_const=100,
                   fixed_point_threshold=1e-20, fixed_point_max_iterations=6, jitter_max_tries=10, explicit=True,
                   softabs=False, jacdiag=False, uniforms=None, seed=0, device=None):
    """Batched samplers.leapfrog with sampler=RMHMC (explicit :389-462 / implicit :305-387), D <= 64.  q, p: (C, D) or
    (D,).  Returns (q_traj (L, C, D), p_traj (L, C, D), q_copy (C, D), p_copy (C, D), failed (C,) uint8)."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    qd, pd = _as_rows(q, ld, device), _as_rows(p, ld, device)
    Cn, L = qd.shape[0], int(steps)
    eps = _eps_vector(step_size, Cn, device)
    cfg = _rmhmc_cfg(D, step_size, jitter, softabs_const, explicit_binding_const, fixed_point_threshold,
                     fixed_point_max_iterations, jitter_max_tries, explicit, softabs, jacdiag)
    keep = []
    rng = _standalone_rng(jitter, uniforms, seed, Cn, D, ld, device, keep)
    q_traj = torch.zeros((L, Cn, ld), dtype=torch.float32, device=device)
    p_traj = torch.zeros_like(q_traj)
    q_copy = torch.zeros((Cn, ld), dtype=torch.float32, device=device)
    p_copy = torch.zeros_like(q_copy)
    failed = torch.zeros(Cn, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_rmhmc_leapfrog(nt.ref(), C.byref(cfg), C.byref(rng), N.ptr(qd), N.ptr(pd), N.ptr(eps), Cn, ld, L,
                                     N.ptr(q_traj), N.ptr(p_traj), N.ptr(q_copy), N.ptr(p_copy), N.ptr(failed),
                                     N.stream_ptr(device))
    N.check(rc, 'hmcx_rmhmc_leapfrog')
    torch.cuda.current_stream(device).synchronize()          # `keep` / the structs may go out of scope now
    return q_traj[..., :D], p_traj[..., :D], q_copy[:, :D], p_copy[:, :D], failed


def rmhmc_hamiltonian(target, q, p, jitter=None, softabs_const=None, softabs=False, jacdiag=False, uniforms=None, seed=0,
                      device=None):
    """Batched rm_hamiltonian (samplers.py:677-736): (H (C,), failed (C,) uint8)."""
    N.require_cuda()
    lib = N.load_library()
    device = torch.device(device if device is not None else (q.device if q.is_cuda else 'cuda'))
    nt = native_target(target, device)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    qd, pd = _as_rows(q, ld, device), _as_rows(p, ld, device)
    Cn = qd.shape[0]
    cfg = _rmhmc_cfg(D, 0.0, jitter, softabs_const, 100, 1e-5, 1, 10, True, softabs, jacdiag)
    keep = []
    rng = _standalone_rng(jitter, uniforms, seed, Cn, D, ld, device, keep)
    H = torch.zeros(Cn, dtype=torch.float32, device=device)
    failed = torch.zeros(Cn, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        rc = lib.hmcx_rmhmc_hamiltonian(nt.ref(), C.byref(cfg), C.byref(rng), N.ptr(qd), N.ptr(pd), Cn, ld, N.ptr(H),
                                        N.ptr(failed), N.stream_ptr(device))
    N.check(rc, 'hmcx_rmhmc_hamiltonian')
    torch.cuda.current_stream(device).synchronize()
    return H, failed


def gemm_nt(A, B):
    """D = A @ B.T on the tensor cores (wgmma) with 3xTF32 split operands (fp32-accurate).  A (M,K), B (N,K) fp32 CUDA;
    M, N multiples of 128, K a multiple of 32."""
    N.require_cuda()
    lib = N.load_library()
    A = A.detach().to(torch.float32).contiguous()
    B = B.detach().to(device=A.device, dtype=torch.float32).contiguous()
    D = torch.empty((A.shape[0], B.shape[0]), dtype=torch.float32, device=A.device)
    with torch.cuda.device(A.device):
        rc = lib.hmcx_gemm_nt_tf32x3(N.ptr(A), N.ptr(B), N.ptr(D), A.shape[0], B.shape[0], A.shape[1],
                                     N.stream_ptr(A.device))
    N.check(rc, 'hmcx_gemm_nt_tf32x3')
    return D

