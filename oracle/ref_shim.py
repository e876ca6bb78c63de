"""TEST INFRASTRUCTURE ONLY -- import the UNMODIFIED reference under sys.modules shims.

The reference (`/root/reference/autoscaler`, pure Python) imports third-party
modules that are absent from this image (pykube, azure-cli, msrestazure,
backports.ssl_match_hostname ...).  None of them performs any arithmetic of the
hot path (SURVEY.md section 8c), so empty stand-ins are enough to import
`autoscaler.cluster`, `autoscaler.scaler`, `autoscaler.engine_scaler`,
`autoscaler.kube`, `autoscaler.capacity` exactly as they lie on disk.

This module only works where the reference tree is present ($ACSFIT_REFERENCE_ROOT, or
the copy oracle/build_ref.py staged in oracle/_ref).  It is used by
`oracle/make_golden*.py` to record the committed fixtures under `tests/golden/`
that the differential tests compare against, and by bench.py's CPU baseline.
Nothing in the product imports it.
"""
import importlib
import json
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))


def _default_root():
    """the reference where it lies in the build container, else the copy oracle/build_ref.py staged in the
    git-ignored oracle/_ref/ (which travels to the GPU box with the snapshot)."""
    if os.path.isdir("/root/reference/autoscaler"):
        return "/root/reference"
    return os.path.join(_HERE, "_ref")


REFERENCE_ROOT = os.environ.get("ACSFIT_REFERENCE_ROOT", _default_root())


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "autoscaler"))


def _mod(name, **attrs):
    m = sys.modules.get(name)
    if m is None:
        m = types.ModuleType(name)
        sys.modules[name] = m
        if "." in name:
            parent, child = name.rsplit(".", 1)
            setattr(_mod(parent), child, m)
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


class _Objects(object):
    """stand-in for pykube's query descriptor: `Pod.objects.namespace = None`
    is assigned at import (cluster.py:21) and `Pod.objects(api)` is called at
    cluster.py:136,157."""
    namespace = None

    def __init__(self):
        self.items = []

    def __call__(self, api):
        return list(self.items)


class _KubeObj(object):
    def __init__(self, api, obj):
        self.api = api
        self.obj = obj

    @property
    def name(self):
        return self.obj["metadata"]["name"]


def install_shims():
    """populate sys.modules with the absent third-party modules."""
    if "pykube" in sys.modules and getattr(sys.modules["pykube"], "_acsfit_shim", False):
        return sys.modules["pykube"]

    class Pod(_KubeObj):
        objects = _Objects()

    class Node(_KubeObj):
        objects = _Objects()

    class HTTPClient(object):
        def __init__(self, config=None):
            self.config = config

    class KubeConfig(object):
        @classmethod
        def from_file(cls, path):
            return cls()

        @classmethod
        def from_service_account(cls):
            return cls()

    class HTTPError(Exception):
        pass

    conn = types.SimpleNamespace(match_hostname=None)
    http = _mod("pykube.http")
    http.requests = types.SimpleNamespace(
        packages=types.SimpleNamespace(urllib3=types.SimpleNamespace(connection=conn)))
    pk = _mod("pykube", Pod=Pod, Node=Node, HTTPClient=HTTPClient, KubeConfig=KubeConfig,
              _acsfit_shim=True)
    _mod("pykube.exceptions", HTTPError=HTTPError)
    _mod("backports")
    _mod("backports.ssl_match_hostname", match_hostname=lambda *a, **k: None)

    def get_file_json(path):
        with open(path) as f:
            return json.load(f)

    class CLIError(Exception):
        pass

    _mod("azure")
    _mod("azure.cli")
    _mod("azure.cli.core")
    _mod("azure.cli.core.util", get_file_json=get_file_json, CLIError=CLIError)
    _mod("azure.cli.core.commands")
    _mod("azure.cli.core.commands.client_factory", get_mgmt_service_client=lambda *a, **k: None)
    _mod("azure.cli.core.azlogging", get_az_logger=lambda *a, **k: None)
    _mod("azure.cli.core.profiles", ResourceType=object)
    _mod("azure.mgmt")
    _mod("azure.mgmt.resource")
    _mod("azure.mgmt.resource.resources", ResourceManagementClient=object)
    _mod("azure.mgmt.compute", ComputeManagementClient=object)
    _mod("azure.mgmt.storage", StorageManagementClient=object)
    _mod("azure.storage")
    _mod("azure.storage.blob", BlockBlobService=object)
    _mod("azure.common", AzureHttpError=Exception)
    _mod("msrestazure")
    _mod("msrestazure.azure_exceptions", CloudError=Exception)
    _mod("msrestazure.azure_operation", AzureOperationPoller=object)
    return pk


def load_reference(capacity_data=None, cpu_reserve=None):
    """returns a namespace with the reference's own modules (unmodified)."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    pk = install_shims()
    os.environ["CAPACITY_DATA"] = capacity_data or os.path.join(REFERENCE_ROOT, "data", "capacity.json")
    if cpu_reserve is not None:
        os.environ["CAPACITY_CPU_RESERVE"] = str(cpu_reserve)
    # drop any previously imported copy so CAPACITY_DATA is re-read (config.py:5)
    for name in [n for n in sys.modules if n == "autoscaler" or n.startswith("autoscaler.")]:
        del sys.modules[name]
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    try:
        ns = types.SimpleNamespace(pykube=pk)
        for short in ("config", "utils", "kube", "capacity", "agent_pool", "scaler",
                      "engine_scaler", "cluster"):
            setattr(ns, short, importlib.import_module("autoscaler." + short))
    finally:
        sys.path.remove(REFERENCE_ROOT)
    return ns
