"""Import-compatibility shim: `from scene_synthesis.networks import build_network` resolves to the
H100-native implementation (diffuscene_b200.networks), so the reference's scripts run unchanged on it."""
