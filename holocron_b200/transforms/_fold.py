"""Run folding shared by the transform chains of the reference's recipes (``segmentation``, ``detection``,
``classification``).

A chain is cut into segments: runs of geometric steps, each folded per image into one ``hb_resample_batch`` row, and
the image-only steps between them. Each image's draws are made for every step in the chain's order before anything is
launched, one image after the other, as the reference's ``Compose`` applied sample by sample makes them."""
from dataclasses import dataclass
from typing import Any, Callable, List, Optional, Sequence, Tuple, Union

from torch import Tensor
from torchvision.transforms import transforms as T
from torchvision.transforms.functional import _compute_resized_output_size

Segment = Union[List[Any], Any]


@dataclass
class _Fold:
    """One image's run folded: its source (the ``box`` = (top, left, height, width) of it when given) resized to
    ``inner``, placed at (top, left) on a canvas of ``canvas``, the canvas mirrored when ``mirror``."""

    inner: Tuple[int, int]
    canvas: Tuple[int, int]
    top: int = 0
    left: int = 0
    mirror: bool = False
    box: Optional[Tuple[int, int, int, int]] = None

    def flip(self) -> None:
        self.mirror = not self.mirror

    def place(self, dy: int, dx: int, h: int, w: int) -> None:
        """The canvas as seen (mirrored or not) moved by (dy, dx) onto a new canvas of h x w: seen pixel (y, x) of the
        new canvas is seen pixel (y - dy, x - dx) of the old one. In a mirrored canvas the placement's columns run the
        other way."""
        self.top += dy
        self.left += (w - self.canvas[1] - dx) if self.mirror else dx
        self.canvas = (h, w)

    def pad(self, bottom: int, right: int) -> None:
        """torchvision's pad of the bottom and right of the canvas."""
        self.place(0, 0, self.canvas[0] + bottom, self.canvas[1] + right)

    def crop(self, i: int, j: int, h: int, w: int) -> None:
        self.place(-i, -j, h, w)

    def center_crop(self, ch: int, cw: int) -> None:
        """torchvision's ``center_crop`` to ch x cw: zero padding where the crop is larger than the canvas, then the
        crop at ``round((H - ch) / 2)``, ``round((W - cw) / 2)`` of the padded canvas."""
        H, W = self.canvas
        pl, pt = max(cw - W, 0) // 2, max(ch - H, 0) // 2
        Hp, Wp = H + pt + max(ch - H + 1, 0) // 2, W + pl + max(cw - W + 1, 0) // 2
        top, left = (0, 0) if (Hp, Wp) == (ch, cw) else (int(round((Hp - ch) / 2.0)), int(round((Wp - cw) / 2.0)))
        self.place(pt - top, pl - left, ch, cw)


def resized(size: Tuple[int, int], out: List[int], max_size: Optional[int] = None) -> Tuple[int, int]:
    """torchvision's output size of a resize of an (H, W) image to ``out``."""
    h, w = _compute_resized_output_size(size, out, max_size)
    return int(h), int(w)


def group(transforms: Sequence[Any], kind: Callable[[Any], Optional[str]], starts_run: Callable[[Any, List[Any]], bool],
          where: str) -> List[Segment]:
    """The steps grouped: runs (lists of geometric steps) and the other steps between them. ``kind(t)`` is "run" for a
    geometric step, "join" for a step that joins an open run and stands alone otherwise, "step" for an image-only step
    and None for what the module does not take; ``starts_run(t, run)`` whether a geometric step opens a new run."""
    segments: List[Segment] = []
    run: Optional[List[Any]] = None
    for t in transforms:
        k = kind(t)
        if k == "join" and run is not None:
            run.append(t)
        elif k == "run":
            if run is None or starts_run(t, run):
                run = []
                segments.append(run)
            run.append(t)
        elif k in ("step", "join"):
            run = None
            segments.append(t)
        else:
            name = getattr(t, "__name__", type(t).__name__)
            raise TypeError(f"{name} is not a transform of holocron_b200.transforms.{where}")
    return segments


def jitters_of(segments: Sequence[Segment], wrapper: type) -> List[Any]:
    """The ``wrapper`` segments around a ColorJitter (torchvision's or this package's)."""
    return [s for s in segments if isinstance(s, wrapper) and isinstance(s.transform, T.ColorJitter)]


def draw(segments: Sequence[Segment], jitters: Sequence[Any], size: Tuple[int, int],
         fold_run: Callable[[Sequence[Any], Tuple[int, int]], _Fold],
         other: Callable[[Any, Tuple[int, int]], Any] = lambda s, size: None) -> List[Any]:
    """One image's draws for every step: the fold of each run, the ``get_params`` of each ColorJitter, ``other(s,
    size)`` for the other steps."""
    plan: List[Any] = []
    for s in segments:
        if isinstance(s, list):
            fold = fold_run(s, size)
            size = fold.canvas
            plan.append(fold)
        elif s in jitters:
            j = s.transform
            plan.append(j.get_params(j.brightness, j.contrast, j.saturation, j.hue))
        else:
            plan.append(other(s, size))
    return plan


def check_stackable(segments: Sequence[Segment], plans: Sequence[Sequence[Any]], sizes: List[Tuple[int, int]],
                    stacks: Callable[[Any], bool] = lambda s: True) -> None:
    """Refuses a step that ``stacks`` the images reached by images of different sizes."""
    for k, s in enumerate(segments):
        if isinstance(s, list):
            sizes = [p[k].canvas for p in plans]
        elif stacks(s) and len(set(sizes)) > 1:
            raise ValueError(f"{s!r} takes images of one size, but the images reaching it have {len(set(sizes))} "
                             "sizes: crop or resize them to one size first")


def sizes_of(images: Sequence[Tensor]) -> List[Tuple[int, int]]:
    return [(int(x.shape[-2]), int(x.shape[-1])) for x in images]
