"""The `.config` of the models and schedulers (no engine import: the schedulers use it on the host)."""
from types import SimpleNamespace


class Config(SimpleNamespace):
    """attribute + mapping access like diffusers' FrozenDict config (`config.scaling_factor`, `config["scaling_factor"]`)"""

    def __getitem__(self, k):
        return getattr(self, k)

    def __contains__(self, k):
        return hasattr(self, k)

    def get(self, k, default=None):
        return getattr(self, k, default)

    def keys(self):
        return self.__dict__.keys()
