import pytest

# pytest rewrites `assert` in test modules only: the shared checks keep their failure detail through this
pytest.register_assert_rewrite("tests.util", "tests.device_cases", "tests.pin_cases")
