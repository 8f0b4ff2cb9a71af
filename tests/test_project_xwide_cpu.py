"""CPU: the projection workspace of the wide Standardized path at 256 < m <= 1024 (csrc/mde_project.cuh).

mde_project_ws_bytes must hold every region of the layout documented above proj_ws_doubles, with each region's size
computed here from that description and from the launch shapes of csrc/mde_project_wide.cu: the tiled Gram writes one
fp32 m x m partial per row block, with 128 x 128 output tiles above m = 256 and 264 / tiles^2 row blocks, at least 16.
The size must grow with m."""
from pymde_b200 import _lib

K_PROJ_BLOCKS = 2 * 132      # kProjBlocks
K_WIDE_ROW_BLOCKS = 2 * 132  # kWideRowBlocks
K_MIN_ROW_BLOCKS = 16        # kWideMinRowBlocks
NEW_WIDTHS = range(257, 1025)


def _row_blocks(m):
    t = 64 if m <= 256 else 128
    tiles = -(-m // t)
    return max(K_WIDE_ROW_BLOCKS // (tiles * tiles), K_MIN_ROW_BLOCKS)


def _regions(m):
    """(name, bytes the kernels use) in layout order; m > 32, so the narrow m x m matrix is empty."""
    mm = m * m
    return [
        ("partials", 8 * K_PROJ_BLOCKS * m),  # column sums of the wide column-mean pass
        ("mean", 8 * m),
        ("shift", 8 * m),
        ("status", 4),
        ("fpart", 4 * _row_blocks(m) * mm),   # the most row blocks a launch uses
        ("gram", 8 * mm),
        ("ns", 8 * 5 * mm),
        ("wf", 4 * mm),
        ("scal", 8 * 4),
        ("nsflag", 4 * 2),
    ]


def _layout_bytes(m):
    """The documented layout: regions in doubles, fp32 regions as (floats / 2 + 1) doubles, the fpart region sized
    max(16 m^2, 264 x 128^2) floats, plus 64 bytes."""
    mm = m * m
    fpart = max(K_MIN_ROW_BLOCKS * mm, K_WIDE_ROW_BLOCKS * 128 * 128)
    doubles = K_PROJ_BLOCKS * m + m + m + 8 + (fpart // 2 + 1) + mm + 5 * mm + (mm // 2 + 1) + 8 + 2
    return 8 * doubles + 64


def test_workspace_holds_every_region_at_every_new_width():
    lib = _lib.load()
    for m in NEW_WIDTHS:
        got = lib.mde_project_ws_bytes(1000, m)
        assert got == _layout_bytes(m), m
        need = sum(b for _, b in _regions(m))
        assert got >= need, "m %d: %d bytes, regions %s" % (m, got, _regions(m))


def test_workspace_grows_with_m():
    lib = _lib.load()
    sizes = [lib.mde_project_ws_bytes(1000, m) for m in range(256, 1025)]
    assert all(b > a for a, b in zip(sizes, sizes[1:]))


def test_workspace_does_not_depend_on_n_and_stays_bounded():
    lib = _lib.load()
    for m in (257, 512, 1024):
        assert lib.mde_project_ws_bytes(3, m) == lib.mde_project_ws_bytes(10 ** 7, m)
    assert lib.mde_project_ws_bytes(1000, 1024) == 123814112  # 118.1 MiB, as mde_project.cuh states
