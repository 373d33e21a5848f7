"""tfservingcache_b200 -- H100-native route -> ensure-resident -> predict path with the API of
mKaloer/TFServingCache.  The product is libtfsc_b200.so (C ABI: include/tfsc_b200.h); this
package is the thin host-side mirror of the reference's Go interfaces over that ABI."""
from . import _lib
from .cluster import ClusterConnection, ReplicaPicker, ServingService, TaskHandler, crc32_ieee, model_key
from .lrucache import LRUCache, Model, ModelIdentifier
from .proxy import RestProxy, GrpcProxy, match_rest_url, parse_version, grpc_model_spec
from .providers import DiskModelProvider
from .server import Server
from .config import load_config
from . import modelformat

__all__ = ["ClusterConnection", "ReplicaPicker", "ServingService", "TaskHandler", "crc32_ieee", "model_key", "LRUCache",
           "Model", "ModelIdentifier", "RestProxy", "GrpcProxy", "match_rest_url", "parse_version",
           "grpc_model_spec", "DiskModelProvider", "Server", "load_config", "modelformat"]
