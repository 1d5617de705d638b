"""h5py is imported at the top of the reference driver (run_pretraining.py:30) and never used on the LDDL path; the real package
is absent offline.  Any attribute access fails loudly."""


def __getattr__(name):
    raise ImportError("h5py stand-in: the HDF5 data path is not part of the H100 hot path (attribute %r requested)" % name)
