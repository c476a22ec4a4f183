"""``dflex.render``: USD export is visualisation only and outside the hot path; the class exists so that
``df.render.UsdRenderer`` resolves, and it fails loudly if actually used without ``pxr``."""


class UsdRenderer:
    def __init__(self, model, stage):
        try:
            import pxr  # noqa: F401
        except ImportError as exc:
            raise ImportError("UsdRenderer needs the `pxr` (usd-core) package, which is not installed; "
                              "construct environments with render=False") from exc
        raise NotImplementedError("USD rendering is not part of the hot-path package")
