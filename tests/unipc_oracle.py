"""Oracle: UniPCMultistepScheduler of diffusers-0.24 (predict_x0, bh1 / bh2), restated the way diffusers writes it:
lists `model_outputs`, `last_sample`, `this_order`, `lower_order_nums`, fp32 torch sigma / lambda arithmetic per step
and torch.linalg.solve for the rhos; no coefficient tables. TEST INFRASTRUCTURE ONLY.

The product (imagdressing_b200/samplers.py) folds every UniPC step into one row of the predictor-corrector kernel;
checking it against this step-by-step formulation checks the table algebra and the slot assignment. The schedule,
add_noise and scale_model_input are DPM-Solver's, so this class reuses DPMSolverOracle's. `oracle.samplers.sample_one`
runs the reference loop with it like with the other oracle schedulers. It lives beside its tests so that the oracle
package, which the other samplers' parity tests measure against, stays as it is.
"""
import torch

from oracle.samplers import DPMSolverOracle


class UniPCOracle(DPMSolverOracle):
    def __init__(self, solver_order=2, solver_type="bh2", lower_order_final=True, disable_corrector=(), **kw):
        super().__init__(solver_order=solver_order, lower_order_final=lower_order_final, **kw)
        self.solver_type, self.disable_corrector = solver_type, list(disable_corrector)

    def set_timesteps(self, n, device=None):
        super().set_timesteps(n, device)
        self.last_sample = None
        self.this_order = None

    def _lambda(self, i):
        alpha, sigma = self._alpha_sigma(self.sigmas[i])
        return alpha, sigma, torch.log(alpha) - torch.log(sigma)

    def _R_b(self, h, rks, order):
        hh = -h
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = hh if self.solver_type == "bh1" else torch.expm1(hh)
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        return h_phi_1, B_h, torch.stack(R), torch.stack(b)

    def _uni_p(self, x, order):
        """multistep_uni_p_bh_update."""
        i = self.step_index
        m0 = self.model_outputs[-1]
        alpha_t, sigma_t, lambda_t = self._lambda(i + 1)
        alpha_s0, sigma_s0, lambda_s0 = self._lambda(i)
        h = lambda_t - lambda_s0
        rks, D1s = [], []
        for k in range(1, order):
            mi = self.model_outputs[-(k + 1)]
            rk = (self._lambda(i - k)[2] - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(torch.tensor(1.0))
        h_phi_1, B_h, R, b = self._R_b(h, torch.stack(rks), order)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        if D1s:
            rhos_p = torch.tensor([0.5]) if order == 2 else torch.linalg.solve(R[:-1, :-1], b[:-1])
            pred_res = sum(r * d for r, d in zip(rhos_p, D1s))
            return x_t_ - alpha_t * B_h * pred_res
        return x_t_

    def _uni_c(self, this_model_output, last_sample, order):
        """multistep_uni_c_bh_update (model_outputs not yet shifted: [-1] is the previous step's)."""
        i = self.step_index
        m0 = self.model_outputs[-1]
        alpha_t, sigma_t, lambda_t = self._lambda(i)
        alpha_s0, sigma_s0, lambda_s0 = self._lambda(i - 1)
        h = lambda_t - lambda_s0
        rks, D1s = [], []
        for k in range(1, order):
            mi = self.model_outputs[-(k + 1)]
            rk = (self._lambda(i - (k + 1))[2] - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(torch.tensor(1.0))
        h_phi_1, B_h, R, b = self._R_b(h, torch.stack(rks), order)
        rhos_c = torch.tensor([0.5]) if order == 1 else torch.linalg.solve(R, b)
        x_t_ = sigma_t / sigma_s0 * last_sample - alpha_t * h_phi_1 * m0
        corr_res = sum(r * d for r, d in zip(rhos_c[:-1], D1s)) if D1s else 0
        D1_t = this_model_output - m0
        return x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * D1_t)

    def step(self, eps, t, x):
        if self.step_index is None:
            self._init_step_index(t)
        i = self.step_index
        use_corrector = i > 0 and i - 1 not in self.disable_corrector and self.last_sample is not None
        alpha_s0, sigma_s0 = self._alpha_sigma(self.sigmas[i])
        m = (x - sigma_s0 * eps) / alpha_s0  # convert_model_output, from the uncorrected sample
        if use_corrector:
            x = self._uni_c(m, self.last_sample, self.this_order)
        self.model_outputs = self.model_outputs[1:] + [m]
        if self.lower_order_final:
            this_order = min(self.solver_order, len(self.timesteps) - i)
        else:
            this_order = self.solver_order
        self.this_order = min(this_order, self.lower_order_nums + 1)
        self.last_sample = x
        out = self._uni_p(x, self.this_order)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return (out,)
