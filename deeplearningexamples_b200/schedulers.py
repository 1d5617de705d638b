"""Device-side learning-rate schedule, mirroring the reference's schedulers.PolyWarmUpScheduler
(PyTorch/LanguageModeling/BERT/schedulers.py:109-136): every quantity is a device tensor so the
training loop stays host-sync free and CUDA-graph capturable; `lr` is *replaced* in each param
group by a fresh 0-dim tensor exactly as the reference does (the optimizer re-reads the pointer).
"""
import torch
from torch.optim.lr_scheduler import _LRScheduler


class PolyWarmUpScheduler(_LRScheduler):
    def __init__(self, optimizer, warmup, total_steps, degree=0.5, last_epoch=-1, base_lr=1., device='cpu'):
        self.warmup = torch.tensor(warmup, device=device)
        self.total_steps = torch.tensor(total_steps, device=device)
        self.degree = torch.tensor(degree, device=device)
        self.base_lr = torch.tensor(base_lr, device=device)
        self.device = device
        # persistent lr scalar: written in place so the optimizer's device tables stay valid
        self._lr_buf = None
        super().__init__(optimizer, torch.tensor(last_epoch, device=device))

    def step(self, epoch=None):
        group0 = self.optimizer.param_groups[0]
        if 'step' in group0:
            self.last_epoch = group0['step'] + 1
        else:
            self.last_epoch = torch.tensor(1., device=self.device)
        for group, lr in zip(self.optimizer.param_groups, self.get_lr()):
            cur = group.get('lr')
            if isinstance(cur, torch.Tensor) and cur.is_cuda and cur.dtype == torch.float32 and cur.dim() == 0:
                cur.copy_(lr.reshape(()))          # same storage => same pointer in the LAMB plan
            else:
                group['lr'] = lr

    def get_lr(self):
        progress = self.last_epoch / self.total_steps
        lr = torch.where(progress < self.warmup, self.base_lr * progress / self.warmup,
                         self.base_lr * ((1.0 - progress) ** self.degree))
        return [lr for _ in self.optimizer.param_groups]


class LinearWarmUpScheduler(_LRScheduler):
    """Linear warm-up to the base rate over `warmup` (a fraction of total_steps), then linear decay to zero at total_steps -- the
    schedule of the SQuAD fine-tuning driver (reference schedulers.py:90-106, used at run_squad.py:1014-1016).
    Host-side by default, like the reference.  With `device` set the schedule is evaluated on the device from the optimizer's own
    step counter (as PolyWarmUpScheduler does), writing the lr tensor in place: no host value is baked into a captured CUDA graph.

    The n-th step (n = 0, 1, ...) runs at progress (n + progress_offset) / total_steps.  The default 1 is the schedule above;
    progress_offset=0 is the SWAG driver's base * warmup_linear(global_step / t_total) (run_swag.py:486-493, optimization.py:46-49),
    whose first step runs at lr 0."""

    def __init__(self, optimizer, warmup, total_steps, last_epoch=-1, device=None, base_lr=None, progress_offset=1):
        self.warmup, self.total_steps = float(warmup), float(total_steps)
        self.progress_offset = float(progress_offset)
        self.device = device
        if device is not None:
            self._base = torch.tensor(float(base_lr if base_lr is not None else 1.0), device=device)
        super().__init__(optimizer, last_epoch)

    def step(self, epoch=None):
        if self.device is not None:
            group0 = self.optimizer.param_groups[0]
            step_t = group0['step'] if isinstance(group0.get('step'), torch.Tensor) else torch.zeros(1, dtype=torch.int32, device=self.device)
            progress = (step_t.reshape(()).float() + self.progress_offset) / self.total_steps
            factor = torch.where(progress < self.warmup, progress / self.warmup,
                                 torch.clamp((progress - 1.0) / (self.warmup - 1.0), min=0.0))
            lr = self._base * factor
            for group in self.optimizer.param_groups:
                cur = group.get('lr')
                if isinstance(cur, torch.Tensor) and cur.is_cuda and cur.dtype == torch.float32 and cur.dim() == 0:
                    cur.copy_(lr)
                else:
                    group['lr'] = lr.clone()
            return
        self.last_epoch = epoch if epoch is not None else self.last_epoch + 1
        for group, lr in zip(self.optimizer.param_groups, self.get_lr()):
            group['lr'] = lr

    def get_lr(self):
        # last_epoch is 0 after construction and n + 1 at the n-th step(); the initial rate is the first step's at offset 0
        progress = max(self.last_epoch - 1.0 + self.progress_offset, 0.0) / self.total_steps
        if progress < self.warmup:
            factor = progress / self.warmup
        else:
            factor = max((progress - 1.0) / (self.warmup - 1.0), 0.0)
        return [base * factor for base in self.base_lrs]
