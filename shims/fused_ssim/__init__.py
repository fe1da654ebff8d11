"""Drop-in for the reference's ``fused_ssim`` package (Reconstruct/submodules/fused-ssim/fused_ssim/__init__.py):
put ``shims/`` on PYTHONPATH ahead of the reference extension and `from fused_ssim import fused_ssim` resolves to
the sm_90a kernels."""
from artdeco_b200.ssim import FusedSSIMMap, allowed_padding, fused_ssim, fusedssim, fusedssim_backward  # noqa: F401
