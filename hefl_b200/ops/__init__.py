"""Python wrappers around the hand-written sm_90a kernels (torch.ops.hefl.*)."""
