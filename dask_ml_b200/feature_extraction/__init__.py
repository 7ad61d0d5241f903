from .text import HashingVectorizer

__all__ = ["HashingVectorizer"]
