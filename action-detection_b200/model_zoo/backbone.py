"""What the engine-backed backbones (BNInception, InceptionV3) share: their convolution and BatchNorm2d children by
attribute name, and the cache of planned engines whose BN-folded weight copies are re-packed when a weight changes."""
from torch import nn


class EngineBackbone(nn.Module):
    """Subclasses fill `_conv_names` and `_bn_names` (the attribute names of each convolution and of its BatchNorm2d, graph
    order) and keep `_engines`, planned engines keyed by everything that shapes their plan."""

    def _convs(self):
        return [getattr(self, n) for n in self._conv_names]

    def _bns(self):
        return [getattr(self, n) for n in self._bn_names]

    def in_channels(self):
        return getattr(self, self._conv_names[0]).in_channels

    def _weights_version(self):
        v = 0
        for c, b in zip(self._convs(), self._bns()):
            v += c.weight._version + c.bias._version + b.weight._version + b.bias._version \
                + b.running_mean._version + b.running_var._version
        return (v, id(self._convs()[0].weight), self._convs()[0].weight.data_ptr())

    def invalidate_packed(self):
        """The kernels read BN-folded, re-laid-out copies of the weights.  They are refreshed automatically when a parameter's
        Tensor._version moves (optimizer.step(), in-place ops); writes that bypass the version counter -- `p.data.copy_()`,
        the fused SGD kernel, a raw pointer -- need this call."""
        for eng in self._engines.values():
            eng.packed_version = None

    def _packed_engine(self, key, make):
        """The engine cached under `key` (make() plans it the first time), its weights packed at their current version."""
        eng = self._engines.get(key)
        if eng is None:
            eng = make()
            self._engines[key] = eng
        ver = self._weights_version()
        if eng.packed_version != ver:
            cs, bs = self._convs(), self._bns()
            eng.pack([c.weight.data for c in cs], [c.bias.data for c in cs], [b.weight.data for b in bs],
                     [b.bias.data for b in bs], [b.running_mean for b in bs], [b.running_var for b in bs])
            eng.packed_version = ver
        return eng
