"""distributed_rl_b200 — H100-native learner-side replay path for
seungju-k1m/Distributed_RL (Ape-X / R2D2 / IMPALA): device-resident sum-tree,
TMA gather, fused target/TD/priority kernels behind the reference's
ReplayMemory / PER / Learner interfaces.  See DESIGN.md."""
__version__ = "0.1.0"
