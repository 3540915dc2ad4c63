"""The work items of a grouped table, restated from the product: what the fused aggregate kernels walk.

build_groups_new (capi.cu) sets seg = clamp(S / (SMs * 64 * 4), 1, 256) series per item, sorts the series by group id with a stable
radix sort (`order`: series ids in group order, ascending ids inside a group) and gives group g ceil(size_g / seg) items of seg
consecutive positions, the last one shorter (group_item_count_kernel, fill_items_kernel in scan_kernels.cu); an empty group has none.
gis[g] is group g's first item.  The fused counter kernel's warp gw takes items gw, gw + nwarps, .. (nwarps = warps * grid), the tile
kernel's CTA c items c, c + grid, .. (scan_wp_ctr.cuh, scan_tile.cuh); merge_partials_kernel's lane j folds a group's items
gis[g] + j, gis[g] + j + 8, .. (scan_kernels.cu)."""
import numpy as np


def seg_for(S, sms):
    """Series per work item of a table of S series on a device of `sms` SMs (scalar tables; histogram tables differ)."""
    return int(min(max(S // (sms * 256), 1), 256))


class Items:
    def __init__(self, groups, G, seg):
        """groups: group id per series (the ungrouped table: all zeros, one group in series order)."""
        groups = np.asarray(groups, np.int64)
        self.S, self.G, self.seg = groups.size, G, seg
        self.order = np.argsort(groups, kind="stable")
        sizes = np.bincount(groups, minlength=G)
        self.group_start = np.concatenate([[0], np.cumsum(sizes)])
        per = (sizes + seg - 1) // seg
        self.gis = np.concatenate([[0], np.cumsum(per)])
        self.n_items = int(self.gis[-1])
        begin = [p for g in range(G) for p in range(self.group_start[g], self.group_start[g + 1], seg)]
        self.item_begin = np.array(begin + [self.S], np.int64)
