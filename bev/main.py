"""``bev.main`` of the reference (simple_romp/bev/main.py): BEV, bev_settings and the lazily evaluated module-level
``default_settings`` (bev/main.py:61), and main(), the ``bev`` command."""
from romp_b200.bev import BEV, bev_settings, main  # noqa: F401

_default = None


def __getattr__(name):
    global _default
    if name == "default_settings":
        if _default is None:
            _default = bev_settings([])
        return _default
    raise AttributeError(name)


if __name__ == "__main__":          # python -m bev.main, like the reference's console script bev=bev.main:main
    main()
