"""``romp.main`` of the reference (simple_romp/romp/main.py): ROMP, romp_settings, main() and the module-level
``default_settings`` (main.py:62: ``romp_settings(input_args=[])``), evaluated on first access instead of at import."""
from romp_b200.main import ROMP, romp_settings, main  # noqa: F401

_default = None


def __getattr__(name):
    global _default
    if name == "default_settings":
        if _default is None:
            _default = romp_settings([])
        return _default
    raise AttributeError(name)


if __name__ == "__main__":          # python -m romp.main, like the reference's console script romp=romp.main:main
    main()
