from .byteTrack.byteTracker import BYTETracker, update_trackers
