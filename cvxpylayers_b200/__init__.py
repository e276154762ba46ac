"""H100-native (sm_90a) batched cone-program solve-and-differentiate engine that plugs in
behind ``cvxpylayers.torch.CvxpyLayer`` in place of the CPU diffcp/SCS path."""
__version__ = "0.1.0"
