"""Helpers shared by the test modules.  No module here is collected by pytest, imports a test module or initialises CUDA on
import."""
