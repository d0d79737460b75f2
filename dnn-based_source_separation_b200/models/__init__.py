"""Drop-in shim: with this directory on PYTHONPATH in place of the reference's src/, ``from models.conv_tasnet import
ConvTasNet`` resolves to the sm_100a implementation (ctn_b200.models.*)."""

# Modules this shim does not provide resolve to the reference's src/ when it follows on sys.path; ours win where both exist.
__path__ = __import__("pkgutil").extend_path(__path__, __name__)
