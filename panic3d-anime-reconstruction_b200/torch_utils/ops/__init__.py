"""sm_90a versions of the StyleGAN custom ops, served under ``torch_utils.ops``: bias_act, upfirdn2d, filtered_lrelu."""
