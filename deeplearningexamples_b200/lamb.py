"""FusedLAMBAMP: drop-in for the reference's lamb_amp_opt.fused_lamb.FusedLAMBAMP, backed by the
three-launch multi-tensor LAMB in libdle_b200.so (csrc/lamb.cu) instead of ~100 launches of
fused_lamb_CUDA.{multi_tensor_l2norm, multi_tensor_lamb}.

Interface mirrored from PyTorch/LanguageModeling/BERT/lamb_amp_opt/fused_lamb/fused_lamb.py:
  ctor kwargs :13-18, device-resident lr/step defaults :21-28 (deep-copied per group, :288-292),
  _step_supports_amp_scaling :39, setup_fp32_params :107-116, zero_grad :118-128,
  step(closure, grad_scaler) :130-260, load_state_dict keeping saved dtype/device :45-105.

Differences (documented in DESIGN.md):
  * 16-bit parameters are bf16 (the reference asserts fp16/fp32, :142); fp32 masters as there.
  * the stage-1 update is never stored -- it is recomputed in fp32 in stage 2 -- whereas the reference
    rounds it to the gradient dtype by writing it into the grad buffer (multi_tensor_lamb.cu:160-170).
    Gradients are therefore left untouched by step().
  * found_inf comes from the same pass that computes the global grad norm (no separate
    GradScaler._check_inf_per_device sweep); the result is registered with the GradScaler so that
    scaler.update() and the driver's `_found_inf_per_device` query (run_pretraining.py:590-592) see it.
"""
import ctypes
from collections import defaultdict
from copy import deepcopy
from itertools import chain

import torch

from . import _lib as L


class FusedLAMBAMP(torch.optim.Optimizer):

    def __init__(self, params, lr=1e-3, step=0, bias_correction=True, betas=(0.9, 0.999), eps=1e-6,
                 weight_decay=0.01, amsgrad=False, adam_w_mode=True, grad_averaging=True, set_grad_none=True,
                 max_grad_norm=1.0, use_nvlamb=False):
        if amsgrad:
            raise RuntimeError('FusedLAMB does not support the AMSGrad variant.')
        if not torch.cuda.is_available():
            raise L.DleError("FusedLAMBAMP needs a CUDA device (no CPU fallback)")
        L.load()
        dev = torch.cuda.current_device()
        defaults = dict(lr=torch.tensor(lr, dtype=torch.float32, device=dev),
                        step=torch.tensor([step], dtype=torch.int, device=dev),
                        bias_correction=bias_correction, betas=betas, eps=eps, weight_decay=weight_decay,
                        grad_averaging=grad_averaging, max_grad_norm=max_grad_norm)
        super().__init__(params, defaults)
        self._step_supports_amp_scaling = True
        self.param_groups_fp32 = []
        self.adam_w_mode = 1 if adam_w_mode else 0
        self.set_grad_none = set_grad_none
        self.use_nvlamb = use_nvlamb
        device = self.param_groups[0]["params"][0].device
        self._dummy_overflow_buf = torch.zeros(1, dtype=torch.int, device=device)
        self._found_inf = torch.zeros(1, dtype=torch.float32, device=device)
        self._global_grad_norm = torch.zeros(1, dtype=torch.float32, device=device)
        self._plan = None
        self._plan_sig = None
        self._lr_dev = []

    def __del__(self):
        self._drop_plan()

    def _drop_plan(self):
        plan = getattr(self, "_plan", None)
        if plan is not None:
            try:
                L.load().dle_lamb_plan_destroy(plan)
            except Exception:
                pass
            self._plan = None
            self._plan_sig = None

    # -- reference API -----------------------------------------------------------------------------
    def add_param_group(self, param_group):
        # tensor-valued defaults (lr, step) must be private to each group (fused_lamb.py:288-292)
        for name, default in self.defaults.items():
            if isinstance(default, torch.Tensor) and name not in param_group:
                param_group[name] = deepcopy(default)
        super().add_param_group(param_group)

    def setup_fp32_params(self):
        """fp32 master copies for 16-bit params (None for fp32 params), fused_lamb.py:107-116."""
        self.param_groups_fp32 = []
        for pg in self.param_groups:
            self.param_groups_fp32.append({'params': [
                p.clone().detach().float() if p.dtype in (torch.bfloat16, torch.float16) else None
                for p in pg['params']]})
        self._drop_plan()

    def zero_grad(self, set_to_none=False):
        for group in self.param_groups:
            for p in group['params']:
                if p.grad is None:
                    continue
                if set_to_none:
                    p.grad = None
                else:
                    if p.grad.grad_fn is not None:
                        p.grad.detach_()
                    else:
                        p.grad.requires_grad_(False)
                    p.grad.zero_()

    def load_state_dict(self, state_dict):
        """Like Optimizer.load_state_dict but state tensors keep the dtype they were saved with
        (fp32 moments for bf16 params) and device-tensor hyper-parameters (lr, step) stay tensors."""
        state_dict = deepcopy(state_dict)
        groups, saved_groups = self.param_groups, state_dict['param_groups']
        if len(groups) != len(saved_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        if any(len(g['params']) != len(s['params']) for g, s in zip(groups, saved_groups)):
            raise ValueError("loaded state dict contains a parameter group that doesn't match the size of optimizer's group")
        id_map = dict(zip(chain.from_iterable(g['params'] for g in saved_groups),
                          chain.from_iterable(g['params'] for g in groups)))

        def to_dev(param, value):
            if isinstance(value, torch.Tensor):
                return value.to(param.device)
            if isinstance(value, dict):
                return {k: to_dev(param, v) for k, v in value.items()}
            return value

        state = defaultdict(dict)
        for k, v in state_dict['state'].items():
            if k in id_map:
                state[id_map[k]] = to_dev(id_map[k], v)
            else:
                state[k] = v
        new_groups = []
        for g, sg in zip(groups, saved_groups):
            dev = g['params'][0].device
            ng = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in sg.items()}
            ng['params'] = g['params']
            new_groups.append(ng)
        self.__setstate__({'state': state, 'param_groups': new_groups})
        self._drop_plan()

    # -- plan construction -------------------------------------------------------------------------
    def _build_plan(self):
        if not self.param_groups_fp32:
            self.setup_fp32_params()
        tensors, groups, grad_dtypes, sig = [], [], set(), []
        for gi, (group, g32) in enumerate(zip(self.param_groups, self.param_groups_fp32)):
            beta1, beta2 = group['betas']
            lg = L.LambGroup()
            # the kernels read lr from a buffer owned by this optimizer: schedulers may REPLACE group['lr'] by a new
            # tensor every step (reference schedulers.py:129-130), which must not invalidate the device tables
            while len(self._lr_dev) <= gi:
                self._lr_dev.append(torch.zeros((), dtype=torch.float32, device=group['params'][0].device))
            if not isinstance(group['step'], torch.Tensor):
                group['step'] = torch.tensor([int(group['step'])], dtype=torch.int, device=group['params'][0].device)
            lg.lr, lg.step = self._lr_dev[gi].data_ptr(), group['step'].data_ptr()
            lg.beta1, lg.beta2, lg.eps, lg.weight_decay = beta1, beta2, group['eps'], group['weight_decay']
            lg.bias_correction = 1 if group['bias_correction'] else 0
            lg.grad_averaging = 1 if group['grad_averaging'] else 0
            groups.append(lg)
            sig.append((group['step'].data_ptr(), beta1, beta2, group['eps'], group['weight_decay']))
            for p, p32 in zip(group['params'], g32['params']):
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError('FusedLAMB does not support sparse gradients')
                if p.dtype not in (torch.float32, torch.bfloat16):
                    raise RuntimeError('FusedLAMBAMP (H100) supports bf16 and fp32 parameters, got %s' % p.dtype)
                if not (p.is_contiguous() and p.grad.is_contiguous()):
                    raise RuntimeError('FusedLAMBAMP needs contiguous parameters and gradients')
                state = self.state[p]
                if len(state) == 0:       # lazily created fp32 moments (fused_lamb.py:215-222)
                    state['exp_avg'] = torch.zeros_like(p.data, dtype=torch.float32)
                    state['exp_avg_sq'] = torch.zeros_like(p.data, dtype=torch.float32)
                for key in ('exp_avg', 'exp_avg_sq'):
                    # load_state_dict keeps whatever dtype a checkpoint held; the kernels take raw fp32 pointers
                    st = state[key]
                    if st.dtype != torch.float32 or st.device != p.device or not st.is_contiguous():
                        state[key] = st.to(device=p.device, dtype=torch.float32).contiguous()
                    if state[key].numel() != p.numel():
                        raise RuntimeError('FusedLAMBAMP: optimizer state %s has %d elements for a parameter of %d'
                                           % (key, state[key].numel(), p.numel()))
                if p32 is not None and (p32.dtype != torch.float32 or p32.device != p.device or not p32.is_contiguous()
                                        or p32.numel() != p.numel()):
                    raise RuntimeError('FusedLAMBAMP: fp32 master copy does not match its parameter; call setup_fp32_params()')
                master = p32 if p.dtype == torch.bfloat16 else p.data
                if p.dtype == torch.bfloat16 and p32 is None:
                    raise RuntimeError('call setup_fp32_params() after casting the model to bf16')
                lt = L.LambTensor()
                lt.grad, lt.param = p.grad.data_ptr(), master.data_ptr()
                lt.exp_avg, lt.exp_avg_sq = state['exp_avg'].data_ptr(), state['exp_avg_sq'].data_ptr()
                lt.model_param = p.data_ptr() if p.dtype == torch.bfloat16 else 0
                lt.numel, lt.group = p.numel(), gi
                tensors.append(lt)
                grad_dtypes.add(p.grad.dtype)
                sig.append((lt.grad, lt.param, lt.exp_avg, lt.exp_avg_sq, lt.model_param, lt.numel))
        if not tensors:
            return None, None
        if len(grad_dtypes) != 1 or next(iter(grad_dtypes)) not in (torch.float32, torch.bfloat16):
            raise RuntimeError('FusedLAMBAMP (H100): all gradients must share one dtype (bf16 or fp32), got %s' % grad_dtypes)
        return (tensors, groups, L.DLE_DTYPE_BF16 if torch.bfloat16 in grad_dtypes else L.DLE_DTYPE_F32), tuple(sig)

    def _grad_signature(self):
        sig = [g['step'].data_ptr() if isinstance(g['step'], torch.Tensor) else -1 for g in self.param_groups]
        for g in self.param_groups:
            for p in g['params']:
                sig.append(p.data_ptr())
                sig.append(p.grad.data_ptr() if p.grad is not None else 0)
        return tuple(sig)

    def _ensure_plan(self):
        gsig = self._grad_signature()
        if self._plan is not None and self._plan_sig is not None and self._plan_sig[0] == gsig:
            return
        built, sig = self._build_plan()
        if built is None:
            self._drop_plan()
            return
        tensors, groups, gdt = built
        tarr = (L.LambTensor * len(tensors))(*tensors)
        shape_sig = (gdt, tuple((t.numel, t.group) for t in tensors),
                     tuple((g.step, g.beta1, g.beta2, g.eps, g.weight_decay, g.bias_correction, g.grad_averaging) for g in groups))
        if self._plan is not None and getattr(self, "_plan_shape_sig", None) == shape_sig:
            # only addresses moved (fresh .grad tensors after zero_grad(set_to_none=True)): patch the device table
            L.check(L.load().dle_lamb_plan_update(self._plan, tarr, len(tensors),
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "dle_lamb_plan_update")
            self._plan_sig = (gsig, sig)
            return
        self._drop_plan()
        self._plan_shape_sig = shape_sig
        garr = (L.LambGroup * len(groups))(*groups)
        plan = ctypes.c_void_p()
        L.check(L.load().dle_lamb_plan_create(tarr, len(tensors), garr, len(groups), gdt, ctypes.byref(plan)),
                "dle_lamb_plan_create")
        self._plan, self._plan_sig = plan, (gsig, sig)
        self._n_plan_tensors = len(tensors)

    # -- step ------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None, grad_scaler=None):
        loss = None
        if closure is not None:
            loss = closure()
        self._ensure_plan()
        device = self.param_groups[0]["params"][0].device
        if self._plan is None:            # no parameter has a gradient: nothing to do, but GradScaler.update() still expects an inf record
            if grad_scaler is not None and grad_scaler.is_enabled():
                self._found_inf.zero_()
                grad_scaler._per_optimizer_states[id(self)]["found_inf_per_device"] = {device: self._found_inf}
            return loss
        for gi, group in enumerate(self.param_groups):
            lr = group['lr']
            if isinstance(lr, torch.Tensor):
                self._lr_dev[gi].copy_(lr.reshape(()), non_blocking=True)
            else:
                self._lr_dev[gi].fill_(float(lr))
        scale = None
        if grad_scaler is not None and grad_scaler.is_enabled():
            scale = grad_scaler._get_scale_async()
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        L.check(L.load().dle_lamb_step(self._plan, ctypes.c_void_p(0 if scale is None else scale.data_ptr()),
                                       float(self.defaults['max_grad_norm']), self.adam_w_mode,
                                       1 if self.use_nvlamb else 0, ctypes.c_void_p(self._found_inf.data_ptr()),
                                       ctypes.c_void_p(self._global_grad_norm.data_ptr()), ctypes.c_void_p(0), stream),
                "dle_lamb_step")
        L.launch_count["n"] += 3
        from . import ops
        ops.weight_epoch["n"] += 1          # parameters changed through raw pointers: invalidate cached bf16 copies
        if grad_scaler is not None and grad_scaler.is_enabled():
            # what GradScaler._check_inf_per_device would have recorded (fused_lamb.py:148-151)
            grad_scaler._per_optimizer_states[id(self)]["found_inf_per_device"] = {device: self._found_inf}
        return loss
