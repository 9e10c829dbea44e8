"""oracle/torch_ema_port.py -- TEST INFRASTRUCTURE, NOT PRODUCT.

Restatement of `torch_ema.ExponentialMovingAverage` (third-party dependency of the reference, imported at nerf/utils.py:29, NOT
vendored in the reference tree and not installed in this image; the reference pins no version -- requirements.txt lists
`torch-ema` bare).  Published algorithm (torch_ema/ema.py of the 0.3 release, the current one when the reference was written):

    __init__(parameters, decay, use_num_updates=True): shadow_params = [p.clone().detach() for p in parameters]; num_updates = 0
    update():   num_updates += 1; decay = min(decay, (1 + num_updates) / (10 + num_updates));
                for s, p: tmp = s - p; tmp *= (1 - decay); s -= tmp
    copy_to():  p.data.copy_(s)          store(): collected = [p.clone()]          restore(): p.data.copy_(collected)
    state_dict(): {"decay", "num_updates", "shadow_params", "collected_params"}

ref_stage.load() registers this module as `torch_ema` when the real package is absent, so that the unmodified reference Trainer
(ema_decay=0.95, main.py:241) runs; tests/ use it as the oracle for the fused EMA kernels (csrc/optim.cu k_ema_update / k_ema_swap).
Parity unpinned against the upstream package itself (absent here); anchored on the reference's call sites (utils.py:544-545,
1213-1214, 1250-1252, 1340-1341, 1364-1365, 1389-1401, 1435-1437).
"""
import torch


class ExponentialMovingAverage:
    def __init__(self, parameters, decay, use_num_updates=True):
        if decay < 0.0 or decay > 1.0:
            raise ValueError("Decay must be between 0 and 1")
        self.decay = decay
        self.num_updates = 0 if use_num_updates else None
        parameters = list(parameters)
        self.shadow_params = [p.clone().detach() for p in parameters]
        self.collected_params = None
        self._params_refs = parameters

    def _get(self, parameters):
        return self._params_refs if parameters is None else list(parameters)

    def update(self, parameters=None):
        parameters = self._get(parameters)
        decay = self.decay
        if self.num_updates is not None:
            self.num_updates += 1
            decay = min(decay, (1 + self.num_updates) / (10 + self.num_updates))
        one_minus_decay = 1.0 - decay
        with torch.no_grad():
            for s_param, param in zip(self.shadow_params, parameters):
                tmp = s_param - param
                tmp.mul_(one_minus_decay)
                s_param.sub_(tmp)

    def copy_to(self, parameters=None):
        for s_param, param in zip(self.shadow_params, self._get(parameters)):
            param.data.copy_(s_param.data)

    def store(self, parameters=None):
        self.collected_params = [p.clone() for p in self._get(parameters)]

    def restore(self, parameters=None):
        if self.collected_params is None:
            raise RuntimeError("This ExponentialMovingAverage has no `store()`ed weights to `restore()`")
        for c_param, param in zip(self.collected_params, self._get(parameters)):
            param.data.copy_(c_param.data)

    def state_dict(self):
        return {"decay": self.decay, "num_updates": self.num_updates, "shadow_params": self.shadow_params,
                "collected_params": self.collected_params}

    def load_state_dict(self, state_dict):
        self.decay = state_dict["decay"]
        self.num_updates = state_dict["num_updates"]
        shadow = state_dict["shadow_params"]
        assert len(shadow) == len(self.shadow_params), "shadow_params must have the same length as the parameters"
        self.shadow_params = [s.to(p.device, p.dtype).clone() for s, p in zip(shadow, self.shadow_params)]
        coll = state_dict.get("collected_params")
        self.collected_params = None if coll is None else [c.clone() for c in coll]
