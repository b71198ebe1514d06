"""pytorch_distributed_b200 - an H100-native (sm_90a, NVLink 4 / NVSwitch) single-node data-parallel training
framework with the capabilities of tczhangzhi/pytorch-distributed (see SURVEY.md / DESIGN.md)."""
__version__ = "0.1.0"
