from .data import MinMaxScaler, RobustScaler, StandardScaler

__all__ = ["StandardScaler", "MinMaxScaler", "RobustScaler"]
