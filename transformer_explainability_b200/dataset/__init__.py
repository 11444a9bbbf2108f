"""Counterpart of the reference's ``dataset`` package: ``install_aliases()`` maps ``dataset.expl_hdf5`` here."""
