"""hotstuff_b200 — H100-native batch Ed25519 verification + SHA-512 digest engine behind the `crypto` crate surface
of asonnino/hotstuff (crypto/src/lib.rs).  Hand-written sm_90a CUDA behind a C ABI (include/hs_crypto.h)."""
from .engine import Engine, EngineError, MultiEngine, VerifyQueue, MODE_STRICT, MODE_BATCH_EQ, bitmap_to_bools  # noqa: F401
from .crypto import CryptoError, Digest, PublicKey, Signature  # noqa: F401
from . import messages, sharding  # noqa: F401,E402  (call-site mirror of consensus/src/messages.rs; multi-GPU sharding)
