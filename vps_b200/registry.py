"""The drop-in boundary: name -> class registries and config-driven builders, without mmcv.

Contract taken from the reference (behaviour, not text): mmdet/utils/registry.py:6-76 -- a registry has `.name`,
`.module_dict`, `.get(key)` (None when absent) and a `register_module` class decorator that refuses non-classes
(TypeError) and duplicate names (KeyError); `build_from_cfg(cfg, registry, default_args)` takes a dict with a `type`
entry (registered name or a class), fills in `default_args` where the config is silent and instantiates;
mmdet/models/registry.py:3-11 names the nine registries; mmdet/models/builder.py:9-45 the build_* helpers
(`build_detector` injects train_cfg / test_cfg, a list of configs becomes an nn.Sequential).

The vps_b200 modules register under the reference's own class names, so configs/cityscapes/fusetrack.py resolves unmodified
here.  `install_into_reference()` is the other integration route SURVEY 8b names: it overwrites the entries of the
REFERENCE's registries (mmdet.models.registry.*.module_dict[name]) with the vps_b200 classes, after which the reference's own
`build_detector` builds the vps_b200 detector from the unmodified config (tests/test_boundary.py).
"""
from torch import nn


class Registry:
    """Ordered table of classes keyed by class name."""

    __slots__ = ("_name", "_table")

    def __init__(self, name):
        self._name = str(name)
        self._table = {}

    # -- the attributes the reference's callers read
    name = property(lambda self: self._name)
    module_dict = property(lambda self: self._table)

    def get(self, key):
        return self._table.get(key)

    def __contains__(self, key):
        return key in self._table

    def __len__(self):
        return len(self._table)

    def __repr__(self):
        return "%s(name=%s, items=%s)" % (type(self).__name__, self._name, list(self._table))

    def register_module(self, cls):
        """Class decorator: `@BACKBONES.register_module`."""
        if not isinstance(cls, type):
            raise TypeError("only classes can be registered in '%s', got %r" % (self._name, type(cls)))
        key = cls.__name__
        if key in self._table:
            raise KeyError("'%s' already holds a class named %s" % (self._name, key))
        self._table[key] = cls
        return cls

    _register_module = register_module      # the reference exposes the undecorated form under this name


def _resolve(kind, registry):
    if isinstance(kind, type):
        return kind
    if isinstance(kind, str):
        cls = registry.get(kind)
        if cls is None:
            raise KeyError("no class named %s in the '%s' registry" % (kind, registry.name))
        return cls
    raise TypeError("cfg['type'] must be a registered name or a class, got %r" % (type(kind),))


def build_from_cfg(cfg, registry, default_args=None):
    if not isinstance(cfg, dict) or "type" not in cfg:
        raise AssertionError("a module config is a dict with a 'type' entry, got %r" % (cfg,))
    if default_args is not None and not isinstance(default_args, dict):
        raise AssertionError("default_args must be a dict or None")
    kwargs = {k: v for k, v in cfg.items() if k != "type"}
    for k, v in (default_args or {}).items():
        kwargs.setdefault(k, v)
    return _resolve(cfg["type"], registry)(**kwargs)


def build(cfg, registry, default_args=None):
    if isinstance(cfg, list):
        return nn.Sequential(*(build_from_cfg(c, registry, default_args) for c in cfg))
    return build_from_cfg(cfg, registry, default_args)


_KINDS = ("backbone", "neck", "extra_neck", "panoptic", "roi_extractor", "shared_head", "head", "loss", "detector")
BACKBONES, NECKS, EXTRA_NECKS, PANOPTIC, ROI_EXTRACTORS, SHARED_HEADS, HEADS, LOSSES, DETECTORS = (Registry(k) for k in _KINDS)
REGISTRIES = dict(BACKBONES=BACKBONES, NECKS=NECKS, EXTRA_NECKS=EXTRA_NECKS, PANOPTIC=PANOPTIC, ROI_EXTRACTORS=ROI_EXTRACTORS,
                  SHARED_HEADS=SHARED_HEADS, HEADS=HEADS, LOSSES=LOSSES, DETECTORS=DETECTORS)


def _maker(registry):
    def make(cfg):
        return build(cfg, registry)
    make.__doc__ = "build a %s from its config dict (or a list of them)" % registry.name
    return make


build_backbone = _maker(BACKBONES)
build_neck = _maker(NECKS)
build_extra_neck = _maker(EXTRA_NECKS)
build_panoptic = _maker(PANOPTIC)
build_roi_extractor = _maker(ROI_EXTRACTORS)
build_shared_head = _maker(SHARED_HEADS)
build_head = _maker(HEADS)
build_loss = _maker(LOSSES)


def build_detector(cfg, train_cfg=None, test_cfg=None):
    return build(cfg, DETECTORS, dict(train_cfg=train_cfg, test_cfg=test_cfg))


def install_into_reference(ref_registry_module):
    """Overwrite the reference's registry entries with the vps_b200 classes of the same name.

    ref_registry_module: the imported `mmdet.models.registry` (it holds BACKBONES ... DETECTORS).  Returns the list of
    (registry, class name) pairs that were replaced or added.  The reference's `register_module` refuses duplicates
    (KeyError), hence the direct `module_dict` assignment -- the route SURVEY 8b describes."""
    done = []
    for attr, mine in REGISTRIES.items():
        theirs = getattr(ref_registry_module, attr, None)
        if theirs is None:
            continue
        for name, cls in mine.module_dict.items():
            theirs.module_dict[name] = cls
            done.append((attr, name))
    return done
