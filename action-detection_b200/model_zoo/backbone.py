"""What the engine-backed backbones (BNInception, InceptionV3) share: their convolution and BatchNorm2d children by
attribute name, the cache of planned engines whose BN-folded weight copies are re-packed when a weight changes, and the
frame count reserved for forward-only engines."""
from torch import nn


class EngineBackbone(nn.Module):
    """Subclasses fill `_conv_names` and `_bn_names` (the attribute names of each convolution and of its BatchNorm2d, graph
    order) and keep `_engines`, planned engines keyed by everything that shapes their plan."""
    _reserved_frames = None

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

    def reserve_frames(self, max_frames):
        """Run every forward-only call of n <= max_frames frames on ONE engine planned for max_frames, with the launches of n
        frames and rows bitwise those of an engine planned for n; a forward of more frames raises.  Without it a model plans,
        allocates and keeps one engine per frame count, which the ragged last chunk of every video multiplies (InceptionV3
        EXACT_TC plans about 106 MB per frame).  Forward-only engines planned per count so far are dropped.  Autograd
        forwards, fused_step and bn_mode='partial' keep their engines per frame count.  max_frames=None goes back to one
        engine per frame count."""
        if max_frames is not None:
            max_frames = int(max_frames)
            if max_frames < 1:
                raise ValueError("reserve_frames: max_frames must be >= 1, got %d" % max_frames)
            for key in [k for k in self._engines if self._forward_only_key(k) and k[0] != max_frames]:
                del self._engines[key]
        self._reserved_frames = max_frames

    def _planned_frames(self, frames, forward_only):
        """the frame count the engine of a call of `frames` frames is planned for"""
        if not forward_only or self._reserved_frames is None:
            return frames
        if frames > self._reserved_frames:
            raise ValueError("a forward of %d frames exceeds the %d frames reserved with reserve_frames(); reserve more or "
                             "split the call" % (frames, self._reserved_frames))
        return self._reserved_frames

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
