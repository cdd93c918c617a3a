"""
Fused multi-tensor Adam: one sm_90a kernel launch updates every parameter tensor of the model
(the reference's torch.optim.Adam, atomai/trainers/trainer.py:539, is ~60 small launches for the
default Unet).  Same update rule, hyper-parameters and state names (`exp_avg`, `exp_avg_sq`,
`step`) as torch.optim.Adam without amsgrad.
"""
import torch

from . import ops


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1:
            raise ValueError("invalid Adam hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._tables = {}
        self.grad_scale = 1.0    # set by the data-parallel trainer to 1/world_size

    def __getstate__(self):
        st = super().__getstate__()
        st = dict(st)
        st["_tables"] = {}        # device pointer tables are never valid in another process
        return st

    def __setstate__(self, state):
        super().__setstate__(state)
        self._tables = {}
        self.__dict__.setdefault("grad_scale", 1.0)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._tables = {}

    def __repr__(self):
        return super().__repr__().replace("FusedAdam", "Adam", 1)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            for p in ps:
                if not p.is_cuda:
                    raise RuntimeError("FusedAdam runs on CUDA (sm_90a) only")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            steps = {int(self.state[p]["step"]) for p in ps}
            assert len(steps) == 1, "parameters of one group must share the step count"
            step = steps.pop() + 1
            key = (gi, tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]["exp_avg"].data_ptr(),
                              self.state[p]["exp_avg_sq"].data_ptr()) for p in ps))
            tab = self._tables.get(gi)
            if tab is None or tab[0] != key:
                rows = []
                for p in ps:
                    assert p.is_contiguous() and p.grad.is_contiguous() and p.dtype == torch.float32
                    st = self.state[p]
                    rows.append([p.data_ptr(), p.grad.data_ptr(), st["exp_avg"].data_ptr(),
                                 st["exp_avg_sq"].data_ptr(), p.numel()])
                tab = (key, torch.tensor(rows, dtype=torch.int64, device=ps[0].device),
                       max(r[4] for r in rows))
                self._tables[gi] = tab
            b1, b2 = group["betas"]
            ops.adam_multi(tab[1], len(ps), tab[2], group["lr"], b1, b2, group["eps"],
                           group["weight_decay"], step, self.grad_scale)
            for p in ps:
                self.state[p]["step"] = step
        return loss
