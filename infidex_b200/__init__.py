"""infidex_b200 -- H100-native (sm_90a) search path behind the lofcz/Infidex API surface."""
from .engine import (Boost, BoostStrength, Document, DocumentFields, Field, NativeError, Query, Result, ScoreEntry, SearchEngine, Stats, Weight)
from .filter import Filter, FilterParseError

__all__ = ["SearchEngine", "Query", "Result", "ScoreEntry", "Document", "DocumentFields", "Field", "Weight", "Filter", "FilterParseError", "Stats", "NativeError", "Boost", "BoostStrength"]
