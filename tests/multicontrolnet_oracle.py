"""fp32 restatement of diffusers-0.24 MultiControlNetModel.forward (pipelines/controlnet/multicontrolnet.py) inside the
reference denoising loop: at step i, net k runs with conditioning_scale = scale_k * keep_k(i) (controlnet_keep,
_controlnet_inpainting.py:373-379,431-436) and the nets' residuals are summed. It plugs into oracle.pipeline.sample_one
and oracle.samplers.sample_one as their `controlnet`, with `control_cond` = the list of per-net images and
control_scale = 1.0 (those loops then pass conditioning_scale = 1.0 at every step)."""


class MultiControlNetOracle:
    def __init__(self, nets, scales, keeps=None):
        """nets: oracle ControlNetModels; scales: one float per net; keeps: None or one 0/1 list per net, one entry per
        step of the loop the oracle is called from."""
        self.nets, self.scales, self.keeps, self.i = list(nets), list(scales), keeps, 0

    def __call__(self, sample, t, text, control_cond, conditioning_scale=1.0):
        down = mid = None
        for k, (net, image, scale) in enumerate(zip(self.nets, control_cond, self.scales)):
            keep = 1.0 if self.keeps is None else self.keeps[k][self.i]
            d, m = net(sample, t, text, image, conditioning_scale=conditioning_scale * scale * keep)
            if down is None:
                down, mid = list(d), m
            else:
                down, mid = [a + b for a, b in zip(down, d)], mid + m
        self.i += 1
        return down, mid


def keep_window(steps, start, end):
    """controlnet_keep of one net over `steps` steps (ipa_controlnet.py:584-590)."""
    return [1.0 - float(i / steps < start or (i + 1) / steps > end) for i in range(steps)]
