"""TEST INFRASTRUCTURE — DPMSolverMultistepScheduler and EulerDiscreteScheduler restated from diffusers 0.24.0
(schedulers/scheduling_dpmsolver_multistep.py, schedulers/scheduling_euler_discrete.py), the version the reference pins
(requirements.txt:5). Kept apart from the product's copies in aniportrait_b200/pipelines/scheduler.py: these are the
scheduler objects the unmodified reference pipeline runs with when make_golden_samplers.py freezes the sampler goldens,
and the ones the oracle loop of the CPU tests steps with.

Restated: `dpmsolver++` / `dpmsolver`, solver_order 1 / 2, `midpoint` / `heun`, lower_order_final, euler_at_final,
Karras sigmas, lambda_min_clipped, every timestep spacing; Euler with its init_noise_sigma, scale_model_input and the
churn-free step. Not restated (they raise): the SDE variants, order 3, thresholding, Euler's s_churn > 0. Neither 0.24
class takes `rescale_betas_zero_snr` or `clip_sample`; `from_config` drops such keys as diffusers' ConfigMixin does."""
from dataclasses import dataclass

import numpy as np
import torch


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas):
    if trained_betas is not None:
        return torch.tensor(trained_betas, dtype=torch.float32)
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    raise NotImplementedError(f"{beta_schedule} is not implemented")


def _sigma_to_t(sigma, log_sigmas):
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(np.shape(sigma))


def _karras(in_sigmas, num_inference_steps, sigma_min=None, sigma_max=None, rho=7.0):
    sigma_min = sigma_min if sigma_min is not None else float(in_sigmas[-1])
    sigma_max = sigma_max if sigma_max is not None else float(in_sigmas[0])
    ramp = np.linspace(0, 1, num_inference_steps)
    min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho


class _FromConfig:
    @classmethod
    def from_config(cls, config, **kwargs):
        """diffusers ConfigMixin.from_config: the keys this class takes, overridden by kwargs; other keys are dropped."""
        import inspect
        names = set(inspect.signature(cls.__init__).parameters) - {"self"}
        cfg = dict(config)
        cfg.update(kwargs)
        return cls(**{k: v for k, v in cfg.items() if k in names})

    def _init_step_index(self, timestep):
        cand = (self.timesteps == timestep).nonzero()
        if len(cand) == 0:
            self._step_index = len(self.timesteps) - 1
        else:
            self._step_index = int(cand[1 if len(cand) > 1 else 0])

    @property
    def step_index(self):
        return self._step_index


@dataclass
class SchedulerOutput:
    prev_sample: torch.Tensor
    pred_original_sample: torch.Tensor = None


class DPMSolverMultistepScheduler(_FromConfig):
    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                 lambda_min_clipped=-float("inf"), variance_type=None, timestep_spacing="linspace", steps_offset=0):
        if algorithm_type not in ("dpmsolver", "dpmsolver++", "sde-dpmsolver", "sde-dpmsolver++"):
            raise NotImplementedError(f"{algorithm_type} is not implemented")
        if solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"{solver_type} is not implemented")
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(
            np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=np.float32)[::-1].copy())
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index = None
        self.config = _Cfg(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                           prediction_type=prediction_type, thresholding=thresholding,
                           dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                           algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
                           euler_at_final=euler_at_final, use_karras_sigmas=use_karras_sigmas,
                           lambda_min_clipped=lambda_min_clipped, variance_type=variance_type,
                           timestep_spacing=timestep_spacing, steps_offset=steps_offset)

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        clipped_idx = torch.searchsorted(torch.flip(self.lambda_t, [0]), c.lambda_min_clipped)
        last_timestep = int(c.num_train_timesteps - clipped_idx)
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, last_timestep - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            step_ratio = last_timestep // (num_inference_steps + 1)
            ts = (np.arange(0, num_inference_steps + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            step_ratio = c.num_train_timesteps / num_inference_steps
            ts = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
            ts -= 1
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported")
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sigmas = np.log(sigmas)
        if c.use_karras_sigmas:
            sigmas = _karras(np.flip(sigmas).copy(), num_inference_steps)
            ts = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas]).round()
            sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(np.float32)
        else:
            sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
            sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
            sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * c.solver_order
        self.lower_order_nums = 0
        self._step_index = None

    @staticmethod
    def _sigma_to_alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def scale_model_input(self, sample, *args, **kwargs):
        return sample

    def convert_model_output(self, model_output, sample):
        c = self.config
        if c.thresholding:
            raise NotImplementedError("dynamic thresholding is not restated")
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(self.sigmas[self.step_index])
        if c.algorithm_type in ("dpmsolver++", "sde-dpmsolver++"):
            if c.prediction_type == "epsilon":
                return (sample - sigma_t * model_output) / alpha_t
            if c.prediction_type == "sample":
                return model_output
            if c.prediction_type == "v_prediction":
                return alpha_t * sample - sigma_t * model_output
        else:
            if c.prediction_type == "epsilon":
                return model_output
            if c.prediction_type == "sample":
                return (sample - alpha_t * model_output) / sigma_t
            if c.prediction_type == "v_prediction":
                return alpha_t * model_output + sigma_t * sample
        raise ValueError(f"prediction_type {c.prediction_type} is not supported")

    def _lambdas(self, *idx):
        out = []
        for i in idx:
            alpha, sigma = self._sigma_to_alpha_sigma_t(self.sigmas[i])
            out.append((alpha, sigma, torch.log(alpha) - torch.log(sigma)))
        return out

    def dpm_solver_first_order_update(self, model_output, sample):
        (alpha_t, sigma_t, lambda_t), (alpha_s, sigma_s, lambda_s) = self._lambdas(self.step_index + 1, self.step_index)
        h = lambda_t - lambda_s
        if self.config.algorithm_type == "dpmsolver++":
            return (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * model_output
        if self.config.algorithm_type == "dpmsolver":
            return (alpha_t / alpha_s) * sample - (sigma_t * (torch.exp(h) - 1.0)) * model_output
        raise NotImplementedError("SDE variants need per-step noise")

    def multistep_dpm_solver_second_order_update(self, model_output_list, sample):
        (alpha_t, sigma_t, lambda_t), (alpha_s0, sigma_s0, lambda_s0), (_, _, lambda_s1) = self._lambdas(
            self.step_index + 1, self.step_index, self.step_index - 1)
        m0, m1 = model_output_list[-1], model_output_list[-2]
        h, h_0 = lambda_t - lambda_s0, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        c = self.config
        if c.algorithm_type == "dpmsolver++":
            if c.solver_type == "midpoint":
                return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                        - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
            return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                    + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1)
        if c.algorithm_type == "dpmsolver":
            if c.solver_type == "midpoint":
                return ((alpha_t / alpha_s0) * sample - (sigma_t * (torch.exp(h) - 1.0)) * D0
                        - 0.5 * (sigma_t * (torch.exp(h) - 1.0)) * D1)
            return ((alpha_t / alpha_s0) * sample - (sigma_t * (torch.exp(h) - 1.0)) * D0
                    - (sigma_t * ((torch.exp(h) - 1.0) / h - 1.0)) * D1)
        raise NotImplementedError("SDE variants need per-step noise")

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, return_dict=True):
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        if self.step_index is None:
            self._init_step_index(timestep)
        c = self.config
        n = len(self.timesteps)
        lower_order_final = (self.step_index == n - 1) and (c.euler_at_final or (c.lower_order_final and n < 15))
        model_output = self.convert_model_output(model_output, sample=sample)
        for i in range(c.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = model_output
        if c.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final:
            prev_sample = self.dpm_solver_first_order_update(model_output, sample=sample)
        elif c.solver_order == 2:
            prev_sample = self.multistep_dpm_solver_second_order_update(self.model_outputs, sample=sample)
        else:
            raise NotImplementedError("solver_order 3 is not restated")
        if self.lower_order_nums < c.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        if not return_dict:
            return (prev_sample,)
        return SchedulerOutput(prev_sample=prev_sample)


class EulerDiscreteScheduler(_FromConfig):
    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, prediction_type="epsilon", interpolation_type="linear", use_karras_sigmas=False,
                 sigma_min=None, sigma_max=None, timestep_spacing="linspace", timestep_type="discrete",
                 steps_offset=0):
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = torch.from_numpy(np.concatenate([sigmas[::-1], [0.0]]).astype(np.float32))
        self.num_inference_steps = None
        timesteps = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy()
        timesteps = torch.from_numpy(timesteps).to(dtype=torch.float32)
        if timestep_type == "continuous" and prediction_type == "v_prediction":
            self.timesteps = torch.Tensor([0.25 * s.log() for s in sigmas])
        else:
            self.timesteps = timesteps
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        self.is_scale_input_called = False
        self.use_karras_sigmas = use_karras_sigmas
        self._step_index = None
        self.config = _Cfg(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                           interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas,
                           sigma_min=sigma_min, sigma_max=sigma_max, timestep_spacing=timestep_spacing,
                           timestep_type=timestep_type, steps_offset=steps_offset)

    @property
    def init_noise_sigma(self):
        max_sigma = self.sigmas.max()
        if self.config.timestep_spacing in ("linspace", "trailing"):
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    def scale_model_input(self, sample, timestep):
        if self.step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self.step_index]
        self.is_scale_input_called = True
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        self.num_inference_steps = num_inference_steps
        n = c.num_train_timesteps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, n - 1, num_inference_steps, dtype=np.float32)[::-1].copy()
        elif c.timestep_spacing == "leading":
            step_ratio = n // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * step_ratio).round()[::-1].copy().astype(np.float32)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            step_ratio = n / num_inference_steps
            ts = (np.arange(n, 0, -step_ratio)).round().copy().astype(np.float32)
            ts -= 1
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported")
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sigmas = np.log(sigmas)
        if c.interpolation_type == "linear":
            sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        elif c.interpolation_type == "log_linear":
            sigmas = torch.linspace(np.log(sigmas[-1]), np.log(sigmas[0]), num_inference_steps + 1).exp().numpy()
        else:
            raise ValueError(f"interpolation_type {c.interpolation_type} is not supported")
        if self.use_karras_sigmas:
            sigmas = _karras(sigmas, self.num_inference_steps, c.sigma_min, c.sigma_max)
            ts = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas])
        sigmas = torch.from_numpy(sigmas).to(dtype=torch.float32)
        if c.timestep_type == "continuous" and c.prediction_type == "v_prediction":
            self.timesteps = torch.Tensor([0.25 * s.log() for s in sigmas]).to(device=device)
        else:
            self.timesteps = torch.from_numpy(ts.astype(np.float32)).to(device=device)
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        self._step_index = None

    def step(self, model_output, timestep, sample, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0,
             generator=None, return_dict=True):
        if isinstance(timestep, int) or (torch.is_tensor(timestep) and not timestep.is_floating_point()):
            raise ValueError("pass one of scheduler.timesteps as the timestep, not an integer index")
        if s_churn > 0:
            raise NotImplementedError("s_churn > 0 needs per-step noise")
        if self.step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self.step_index]
        pt = self.config.prediction_type
        if pt in ("original_sample", "sample"):
            x0 = model_output
        elif pt == "epsilon":
            x0 = sample - sigma * model_output
        elif pt == "v_prediction":
            x0 = model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))
        else:
            raise ValueError(f"prediction_type {pt} is not supported")
        derivative = (sample - x0) / sigma
        dt = self.sigmas[self.step_index + 1] - sigma
        prev_sample = sample + derivative * dt
        self._step_index += 1
        if not return_dict:
            return (prev_sample,)
        return SchedulerOutput(prev_sample=prev_sample, pred_original_sample=x0)
