"""gps-gaussian_b200: H100-native (sm_90a) splat rasterizer + 1-D stereo correlation sampler
behind GPS-Gaussian's own call signatures (reference gaussian_renderer/__init__.py:17,
lib/GaussianRender.py:5, core/corr.py:17-61).  See DESIGN.md."""
__version__ = "0.1.0"
