"""What the host side of every resident table (gp_*_table_* of include/gangpack.h) does the same way: its capacities, the
replay that resets the device's table and resends the whole state, and flush(), which delivers one delta to a packer."""
from __future__ import annotations


class ResidentTable:
    """The base of reservations.ReservationTable, overhead.OverheadTable, affinity.LabelTable, nodes.NodeTable and
    drivers.DriverTable.  A subclass sets `name` (the packer's <name>_table_reset and <name>_table_update) and `writes` (the
    delta arrays whose lengths count its writes), and gives

        _bounds()          {size key: the least capacity the state needs}
        _changes(replay)   the arrays of one update: every row (replay true) or what changed since the last delta; the
                           changes count as sent

    delta() -> the arrays of one update.  When it carries "reset" (the first one, whenever a capacity would be exceeded: it is
    doubled and the whole state replayed, and after replay()), the <name>_table_reset(**delta["reset"]) goes first.
    `replays` counts the deltas that carry one; `mirror` is a numpy copy of what the device holds, kept by flush()."""

    name = None
    writes = ()

    def __init__(self, mirror, **size):
        self.size = size
        self.mirror = mirror
        self._replay = True
        self.replays = 0

    def replay(self):
        """The next delta resets the table and resends the whole state.  delta() takes its changes as sent, so after an
        update the library refused or that failed, call this: otherwise the host and the device disagree for good."""
        self._replay = True

    def delta(self) -> dict:
        for k, b in self._bounds().items():
            while self.size[k] < b:
                self.size[k] = max(2 * self.size[k], 1)
                self._replay = True
        if self._replay:
            self.replays += 1
        d = {"reset": dict(self.size) if self._replay else None, **self._changes(self._replay)}
        self._replay = False
        return d

    def flush(self, packer):
        """One update of the device's table (none when nothing changed), preceded by a reset when the delta carries one; on
        a refusal the whole state is reset and replayed once more, and a second refusal is raised."""
        from .native import GangpackError
        d = self.delta()
        if d["reset"] is None and not any(len(d[k]) for k in self.writes):
            return
        try:
            self.push(packer, d)
        except GangpackError:
            self.replay()
            d = self.delta()
            self.push(packer, d)
        self.mirror.apply(d)

    def push(self, packer, d):
        """Deliver delta d: the reset it carries, then the update.  flush() delivers the table's own deltas; a caller that
        takes them with delta() itself delivers each with this."""
        if d["reset"] is not None:
            getattr(packer, f"{self.name}_table_reset")(**d["reset"])
        getattr(packer, f"{self.name}_table_update")(d)
