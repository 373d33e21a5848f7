"""Restatement of the reference's residency state machine (CPU oracle, pure Python).

Follows:
  pkg/cachemanager/cachemanager.go:91-152   fetchModel: hit / cached-but-unloaded / miss
  pkg/cachemanager/cachemanager.go:154-165  tryGetModelFromCache (LRU.Get touches recency)
  pkg/cachemanager/cachemanager.go:167-195  reloadServingConfig: resident := first
                                             min(len, maxConcurrentModels) of the MRU list
  pkg/cachemanager/servingcontroller.go:29-54   ModelVersionStatus_State enum
  pkg/cachemanager/servingcontroller.go:159-187 createModelConfig (group by name, first seen)

Tier mapping used by the GPU build (DESIGN.md): the reference's on-disk LRU
(``modelCache.size`` bytes) is the *pinned-host tier*; "loaded in TF-Serving"
(``serving.maxConcurrentModels``) is the *HBM-resident tier*, additionally bounded by the HBM
arena byte budget.  TF-Serving is restated as ``_Serving``: after a reload exactly the pushed
set is AVAILABLE, everything previously loaded and no longer listed is END.
The reference's outcome per request is one of "hit" | "reload" | "miss"; hits are the only
branch that increments cache_hits_total, misses the only one that increments
cache_misses_total (cachemanager.go:103-150).
"""
from __future__ import annotations

from .lrucache import LRUCache, Model, ModelIdentifier

UNKNOWN, START, LOADING, AVAILABLE, UNLOADING, END = 0, 10, 20, 30, 40, 50


class ModelNotFound(Exception):
    """GetModelStatus: len(resp.ModelVersionStatus)==0 -> errors.New("Model not found")."""


class _Serving:
    def __init__(self):
        self.state: dict[ModelIdentifier, int] = {}

    def reload(self, models: list[Model]):
        wanted = [m.identifier for m in models]
        loaded, unloaded = [], []
        for ident, st in list(self.state.items()):
            if st == AVAILABLE and ident not in wanted:
                self.state[ident] = END
                unloaded.append(ident)
        for ident in wanted:
            if self.state.get(ident) != AVAILABLE:
                self.state[ident] = AVAILABLE
                loaded.append(ident)
        return loaded, unloaded

    def status(self, ident: ModelIdentifier) -> int:
        if ident not in self.state:
            raise ModelNotFound("Model not found")
        return self.state[ident]


class CacheManager:
    def __init__(self, provider, cache_bytes: int, max_concurrent_models: int,
                 arena_bytes: int | None = None):
        self.provider = provider  # .model_size(name, ver) / .load_model(name, ver) -> Model
        self.local_cache = LRUCache("", cache_bytes)
        self.max_concurrent_models = max_concurrent_models
        self.arena_bytes = arena_bytes
        self.serving = _Serving()
        self.total = self.hits = self.misses = 0
        self.log: list[tuple] = []  # (outcome, ident, loaded, unloaded, host_evicted)

    def resident_prefix(self) -> list[Model]:
        avail = self.local_cache.list_models()
        n = min(len(avail), self.max_concurrent_models)
        active = avail[:n]
        if self.arena_bytes is not None:  # HBM byte budget (new-build addition)
            out, used = [], 0
            for m in active:
                if used + m.size_on_disk > self.arena_bytes:
                    break
                out.append(m)
                used += m.size_on_disk
            active = out
        return active

    def _reload(self):
        return self.serving.reload(self.resident_prefix())

    def fetch_model(self, ident: ModelIdentifier) -> str:
        self.total += 1
        n_ev = len(self.local_cache.evicted)
        model, present = self.local_cache.get(ident)
        loaded = unloaded = ()
        if not present:
            self.misses += 1
            size = self.provider.model_size(ident.model_name, ident.version)
            self.local_cache.ensure_free_bytes(size)
            model = self.provider.load_model(ident.model_name, ident.version)
            self.local_cache.put(ident, model)
            # new-build fix: a model dropped from the host tier leaves HBM immediately
            for ev in self.local_cache.evicted[n_ev:]:
                if self.serving.state.get(ev) == AVAILABLE:
                    self.serving.state[ev] = END
            loaded, unloaded = self._reload()
            outcome = "miss"
        else:
            try:
                st = self.serving.status(ident)
                need = st in (UNLOADING, END)
            except ModelNotFound:
                need = True
            if need:
                loaded, unloaded = self._reload()
                outcome = "reload"
            else:
                self.hits += 1
                outcome = "hit"
        self.log.append((outcome, ident, tuple(loaded), tuple(unloaded),
                         tuple(self.local_cache.evicted[n_ev:])))
        return outcome

    def handle_model_request(self, model_name: str, version: str) -> str:
        from .urlmatch import parse_version
        return self.fetch_model(ModelIdentifier(model_name, parse_version(version)))


def create_model_config(models: list[Model], serving_model_dir: str) -> list[dict]:
    """servingcontroller.go:159-187."""
    distinct: dict[str, dict] = {}
    configs: list[dict] = []
    for m in models:
        name = m.identifier.model_name
        if name in distinct:
            distinct[name]["versions"].append(m.identifier.version)
        else:
            cfg = {"name": name, "base_path": serving_model_dir.rstrip("/") + "/" + name,
                   "model_platform": "tensorflow", "versions": [m.identifier.version]}
            distinct[name] = cfg
            configs.append(cfg)
    return configs
